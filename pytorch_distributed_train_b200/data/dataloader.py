"""DataLoader for the single-process-per-GPU input path of the reference
(ref: ddp_example.py:73-78: ``batch_size=100, shuffle=False, num_workers=0, pin_memory=True,
sampler=train_sampler``; torch/utils/data/dataloader.py:773-805 for the contract:
BatchSampler → fetch → collate → pin).

H100-first changes (the host must keep a ~0.1 ms training step fed):

* **batched gather**: datasets that expose ``gather(indices) -> tuple[Tensor, ...]`` (our MNIST and
  synthetic datasets do) are sliced with one ``index_select`` per field instead of a Python loop
  over samples plus ``default_collate`` (the reference pays 100 PIL round trips per step here);
* **pinned batches**: every batch is copied into a fresh pinned tensor from torch's event-tracked caching host
  allocator (a free-list pop after warm-up), so a consumer that runs ahead of the GPU can never see a batch
  overwritten under a pending H2D copy;
* **native stager**: tensor-backed datasets (``native_source()``: MNIST, SyntheticMNIST) are batched by a C++ worker
  thread (``_C.BatchStager``) that gathers the sampler's order, applies ToTensor's 1/255 and writes into a ring of
  pinned buffers allocated once; a slot is reused only after the consumer's H2D copies out of it have completed (CUDA
  event) and nobody holds the batch any more;
* **prefetch thread**: optional background producer (``prefetch=k``) so batch *i+1* is being
  assembled while step *i* runs;
* :class:`DevicePrefetcher` overlaps the H2D copy of batch *i+1* with compute of batch *i* on a
  dedicated copy stream.
"""
from __future__ import annotations

import queue
import threading
from typing import Any, Callable, Iterator, List, Optional, Sequence

import torch

from .sampler import BatchSampler, RandomSampler, SequentialSampler


def _native_mod():
    from .. import _C

    return _C


def default_collate(batch: Sequence[Any]):
    elem = batch[0]
    if isinstance(elem, torch.Tensor):
        return torch.stack(list(batch), 0)
    if isinstance(elem, (int, bool)):
        return torch.tensor(batch, dtype=torch.int64)
    if isinstance(elem, float):
        return torch.tensor(batch, dtype=torch.float64)
    if isinstance(elem, (tuple, list)):
        return type(elem)(default_collate(s) for s in zip(*batch)) if isinstance(elem, tuple) else [default_collate(s) for s in zip(*batch)]
    if isinstance(elem, dict):
        return {k: default_collate([d[k] for d in batch]) for k in elem}
    try:
        import numpy as np

        if isinstance(elem, np.ndarray):
            return torch.stack([torch.from_numpy(b) for b in batch], 0)
        if isinstance(elem, np.generic):
            return torch.tensor(batch)
    except ImportError:  # pragma: no cover
        pass
    raise TypeError(f"default_collate: unsupported element type {type(elem)}")


def _map_tensors(obj, fn):
    if isinstance(obj, torch.Tensor):
        return fn(obj)
    if isinstance(obj, tuple):
        return tuple(_map_tensors(o, fn) for o in obj)
    if isinstance(obj, list):
        return [_map_tensors(o, fn) for o in obj]
    if isinstance(obj, dict):
        return {k: _map_tensors(v, fn) for k, v in obj.items()}
    return obj


_WARM_POOL: set = set()
_WARM_BLOCKS = 24


def _pin_batch(batch):
    """Copy a batch into *fresh* pinned tensors from torch's caching host allocator.

    Fresh, not a private ring: the consumer issues ``.to(device, non_blocking=True)`` (ref: ddp_example.py:83-84) and
    may run many batches ahead of the GPU (a graph-replayed step is ~0.1 ms).  The caching host allocator records a
    CUDA event for every non-blocking copy out of a pinned block and recycles the block only after that event has
    completed, so a batch can never be overwritten while its H2D copy is still pending — and two batches of one
    ``list(loader)`` never alias.  After warm-up an allocation is a free-list pop (no ``cudaHostAlloc``)."""
    if not torch.cuda.is_available():
        return batch

    def pin(t: torch.Tensor):
        if t.is_pinned():
            return t
        sig = (tuple(t.shape), t.dtype)
        if sig not in _WARM_POOL:
            # Pre-warm the allocator's free list for this batch signature: a pool miss later means cudaHostAlloc, which
            # was measured stalling the loader for tens of milliseconds in the middle of a run.  A block
            # is recycled only after the H2D copy out of it has completed, so a consumer that runs several steps ahead of
            # the GPU keeps a dozen blocks of each kind in flight.
            _WARM_POOL.add(sig)
            warm = [torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for _ in range(_WARM_BLOCKS)]
            del warm
        buf = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
        buf.copy_(t)
        return buf

    return _map_tensors(batch, pin)


class DataLoader:
    def __init__(self, dataset, batch_size: Optional[int] = 1, shuffle: bool = False, sampler=None,
                 batch_sampler=None, num_workers: int = 0, collate_fn: Optional[Callable] = None,
                 pin_memory: bool = False, drop_last: bool = False, prefetch: int = 0,
                 generator: Optional[torch.Generator] = None, native: Optional[bool] = None):
        if num_workers != 0:
            # worker *processes* are not needed for tensor-backed datasets; a thread prefetcher is
            # what keeps up with a graph-replayed step. Map the knob instead of failing.
            prefetch = max(prefetch, 2 * num_workers)
        if sampler is not None and shuffle:
            raise ValueError("sampler option is mutually exclusive with shuffle")
        if batch_sampler is not None and (batch_size not in (1, None) or shuffle or sampler is not None or drop_last):
            raise ValueError("batch_sampler option is mutually exclusive with batch_size, shuffle, sampler, and drop_last")
        own_batching = batch_sampler is None   # the loader batches the sampler itself (a user batch_sampler owns the grouping)
        self.dataset = dataset
        self.batch_size = batch_size
        self.drop_last = drop_last
        self.pin_memory = pin_memory
        self.collate_fn = collate_fn
        self.prefetch = prefetch
        if batch_sampler is None:
            if sampler is None:
                sampler = RandomSampler(dataset, generator) if shuffle else SequentialSampler(dataset)
            batch_sampler = BatchSampler(sampler, batch_size, drop_last) if batch_size is not None else None
        self.sampler = sampler
        self.batch_sampler = batch_sampler
        self._can_gather = collate_fn is None and hasattr(dataset, "gather")
        # native path: a C++ worker thread stages batches into a pinned ring (no GIL, no intra-op thread pool, no
        # allocator traffic in steady state); needs a tensor-backed dataset and the default collation
        self._native = None
        self._native_src = None
        if collate_fn is None and own_batching and self.batch_size is not None and hasattr(dataset, "native_source") and native is not False:
            src = dataset.native_source()
            if src is not None and hasattr(_native_mod(), "BatchStager"):
                self._native_src = src
        if native is True and self._native_src is None:
            raise ValueError("DataLoader(native=True) needs a dataset with native_source() and the default collate_fn / batch sampler")

    def __len__(self) -> int:
        return len(self.batch_sampler) if self.batch_sampler is not None else len(self.sampler)

    def _fetch(self, indices: List[int]):
        if self._can_gather:
            batch = self.dataset.gather(indices)
        else:
            samples = [self.dataset[i] for i in indices]
            batch = (self.collate_fn or default_collate)(samples)
        if self.pin_memory:
            batch = _pin_batch(batch)
        return batch

    def _iter_sync(self) -> Iterator:
        if self.batch_sampler is None:
            for i in self.sampler:
                yield self.dataset[i]
            return
        for indices in self.batch_sampler:
            yield self._fetch(indices)

    def _iter_prefetch(self) -> Iterator:
        q: "queue.Queue" = queue.Queue(maxsize=self.prefetch)
        stop = threading.Event()
        END = object()

        def produce():
            try:
                for indices in self.batch_sampler:
                    if stop.is_set():
                        return
                    q.put(self._fetch(indices))
                q.put(END)
            except BaseException as e:  # noqa: BLE001 - forwarded to the consumer
                q.put(e)

        th = threading.Thread(target=produce, name="pdt-dataloader", daemon=True)
        th.start()
        try:
            while True:
                item = q.get()
                if item is END:
                    return
                if isinstance(item, BaseException):
                    raise item
                yield item
        finally:
            stop.set()
            while th.is_alive():
                try:
                    q.get_nowait()
                except queue.Empty:
                    th.join(0.01)

    def _iter_native(self) -> Iterator:
        src = self._native_src
        if self._native is None:
            pin = bool(self.pin_memory and torch.cuda.is_available())
            dev = torch.cuda.current_device() if pin else -1
            self._native = _native_mod().BatchStager(src["data"], src["targets"], list(src["sample_shape"]), int(self.batch_size),
                                                     bool(self.drop_last), float(src["scale"]), max(8, self.prefetch + 4), pin, dev)
        # the sampler decides the epoch's order, once (tensor fast path: no 60,000-element Python list per epoch)
        order = self.sampler.indices_tensor() if hasattr(self.sampler, "indices_tensor") else torch.as_tensor(list(iter(self.sampler)), dtype=torch.int64)
        self._native.start(order)
        while True:
            item = self._native.next()
            if item is None:
                return
            yield item

    def __iter__(self) -> Iterator:
        if self._native_src is not None:
            return self._iter_native()
        if self.prefetch > 0 and self.batch_sampler is not None:
            return self._iter_prefetch()
        return self._iter_sync()


class DevicePrefetcher:
    """Wraps a loader; yields device tensors, with the H2D copy of the next batch overlapped on a
    side stream (pinned source ⇒ truly asynchronous). Equivalent of the reference's
    ``images.cuda(non_blocking=True)`` (ref: ddp_example.py:83-84) but one batch ahead."""

    def __init__(self, loader, device):
        self.loader = loader
        self.device = torch.device(device)
        self.stream = torch.cuda.Stream(device=self.device) if self.device.type == "cuda" else None

    def __len__(self):
        return len(self.loader)

    def __iter__(self):
        if self.stream is None:
            yield from self.loader
            return
        it = iter(self.loader)

        def load():
            try:
                b = next(it)
            except StopIteration:
                return None
            with torch.cuda.stream(self.stream):
                return _map_tensors(b, lambda t: t.to(self.device, non_blocking=True))

        nxt = load()
        while nxt is not None:
            torch.cuda.current_stream(self.device).wait_stream(self.stream)
            cur = nxt
            _map_tensors(cur, lambda t: t.record_stream(torch.cuda.current_stream(self.device)) or t)
            nxt = load()
            yield cur
