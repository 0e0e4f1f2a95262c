"""Samplers. ``DistributedSampler`` reproduces the index semantics the reference relies on
(ref: ddp_example.py:70-72 → torch/utils/data/distributed.py:17-157): per-epoch seeded
permutation shared by all replicas, wrap-around padding (or truncation with ``drop_last``) to a
multiple of the replica count, then a strided slice ``indices[rank::num_replicas]``.

The permutation itself comes from ``torch.randperm`` with a ``torch.Generator`` seeded
``seed + epoch`` so shards are bit-identical to the reference's for the same arguments.
"""
from __future__ import annotations

import math
from typing import Iterator, List, Optional, Sized

import torch


class Sampler:
    def __iter__(self) -> Iterator[int]:
        raise NotImplementedError


class SequentialSampler(Sampler):
    def __init__(self, data_source: Sized):
        self.data_source = data_source

    def __iter__(self):
        return iter(range(len(self.data_source)))

    def __len__(self):
        return len(self.data_source)


class RandomSampler(Sampler):
    def __init__(self, data_source: Sized, generator: Optional[torch.Generator] = None):
        self.data_source = data_source
        self.generator = generator

    def __iter__(self):
        g = self.generator
        if g is None:
            g = torch.Generator()
            g.manual_seed(int(torch.empty((), dtype=torch.int64).random_().item()))
        return iter(torch.randperm(len(self.data_source), generator=g).tolist())

    def __len__(self):
        return len(self.data_source)


class BatchSampler(Sampler):
    def __init__(self, sampler, batch_size: int, drop_last: bool):
        if batch_size <= 0:
            raise ValueError(f"batch_size should be a positive integer, got {batch_size}")
        self.sampler, self.batch_size, self.drop_last = sampler, batch_size, drop_last

    def __iter__(self) -> Iterator[List[int]]:
        batch: List[int] = []
        for idx in self.sampler:
            batch.append(idx)
            if len(batch) == self.batch_size:
                yield batch
                batch = []
        if batch and not self.drop_last:
            yield batch

    def __len__(self):
        n = len(self.sampler)
        return n // self.batch_size if self.drop_last else (n + self.batch_size - 1) // self.batch_size


class DistributedSampler(Sampler):
    def __init__(self, dataset: Sized, num_replicas: Optional[int] = None, rank: Optional[int] = None,
                 shuffle: bool = True, seed: int = 0, drop_last: bool = False):
        if num_replicas is None or rank is None:
            from .. import distributed as dist

            if not dist.is_initialized():
                raise RuntimeError("DistributedSampler needs num_replicas and rank, or an initialised process group")
            num_replicas = dist.get_world_size() if num_replicas is None else num_replicas
            rank = dist.get_rank() if rank is None else rank
        if rank >= num_replicas or rank < 0:
            raise ValueError(f"Invalid rank {rank}, rank should be in the interval [0, {num_replicas - 1}]")
        self.dataset = dataset
        self.num_replicas = num_replicas
        self.rank = rank
        self.epoch = 0
        self.drop_last = drop_last
        n = len(dataset)
        if drop_last and n % num_replicas != 0:
            self.num_samples = math.ceil((n - num_replicas) / num_replicas)
        else:
            self.num_samples = math.ceil(n / num_replicas)
        self.total_size = self.num_samples * num_replicas
        self.shuffle = shuffle
        self.seed = seed

    def _global_order(self) -> List[int]:
        n = len(self.dataset)
        if self.shuffle:
            g = torch.Generator()
            g.manual_seed(self.seed + self.epoch)
            order = torch.randperm(n, generator=g).tolist()
        else:
            order = list(range(n))
        if not self.drop_last:
            pad = self.total_size - len(order)
            if pad > 0:
                if pad <= len(order):
                    order += order[:pad]
                else:  # dataset smaller than the padding: wrap as often as needed
                    order += (order * math.ceil(pad / len(order)))[:pad]
        else:
            order = order[: self.total_size]
        return order

    def __iter__(self) -> Iterator[int]:
        order = self._global_order()
        shard = order[self.rank: self.total_size: self.num_replicas]
        assert len(shard) == self.num_samples
        return iter(shard)

    def indices_tensor(self) -> torch.Tensor:
        """This rank's indices of the current epoch as an int64 tensor — the same sequence ``__iter__`` yields, built with tensor ops
        only (60,000 Python ints cost milliseconds per epoch start, many training steps of the reference ConvNet) and cached while
        (seed, epoch) do not change: the reference never calls ``set_epoch``, so every epoch after the first restarts for free."""
        n = len(self.dataset)
        key = (self.seed, self.epoch, self.shuffle, n, self.num_replicas, self.rank, self.drop_last)
        if getattr(self, "_order_key", None) == key:
            return self._order_cache
        if self.shuffle:
            g = torch.Generator()
            g.manual_seed(self.seed + self.epoch)
            order = torch.randperm(n, generator=g)
        else:
            order = torch.arange(n, dtype=torch.int64)
        if not self.drop_last:
            pad = self.total_size - n
            if pad > 0:
                reps = math.ceil(pad / max(n, 1))
                order = torch.cat([order, order.repeat(reps)[:pad]])
        else:
            order = order[: self.total_size]
        shard = order[self.rank: self.total_size: self.num_replicas].contiguous()
        assert shard.numel() == self.num_samples
        self._order_key, self._order_cache = key, shard
        return shard

    def __len__(self) -> int:
        return self.num_samples

    def set_epoch(self, epoch: int) -> None:
        """Call at the start of each epoch for a different shuffle; the reference never does
        (ref: ddp_example.py:81), which is why it sees the same order every epoch."""
        self.epoch = epoch
