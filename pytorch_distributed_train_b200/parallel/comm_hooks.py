"""Gradient communication hooks for :class:`DistributedDataParallel`.

Interface parity: ``ddp.register_comm_hook(state, hook)`` with
``hook(state, bucket: GradBucket) -> Future[Tensor]`` (torch c10d comm.hpp:20-118,
ddp_comm_hooks/default_hooks.py:35-175).  The bucket a hook receives holds *undivided* local
gradients (observed behaviour of the reference stack); the hook owns the
averaging.  The reference script itself installs no hook (ref: ddp_example.py:64) — the built-in
path is the fused reduce kernel — so these are the optional surface.
"""
from __future__ import annotations

from typing import Callable, List, Optional

import torch

from .. import distributed as dist


class Future:
    """Minimal future: a value that becomes available after a collective's ``wait()``."""

    def __init__(self, work=None, value: Optional[torch.Tensor] = None):
        self._work = work
        self._value = value
        self._callbacks: List[Callable] = []
        self._done = work is None

    def then(self, fn: Callable[["Future"], torch.Tensor]) -> "Future":
        self._callbacks.append(fn)
        return self

    def wait(self) -> torch.Tensor:
        if not self._done:
            self._work.wait()
            self._done = True
        for fn in self._callbacks:
            self._value = fn(self)
        self._callbacks = []
        return self._value

    def value(self) -> torch.Tensor:
        return self.wait()

    def done(self) -> bool:
        return self._done or self._work.is_completed()


def _group(state):
    return state if isinstance(state, dist.ProcessGroup) else dist.get_default_group()


def allreduce_hook(state, bucket) -> Future:
    """Average gradients: sum-allreduce with the 1/world scale folded into the collective."""
    g = _group(state)
    buf = bucket.buffer()
    return Future(g.comm.allreduce(buf, dist.ReduceOp.SUM, 1.0 / g.size()), buf)


def _compress_hook(dtype):
    def hook(state, bucket) -> Future:
        g = _group(state)
        buf = bucket.buffer()
        wire = buf.to(dtype).div_(g.size())
        fut = Future(g.comm.allreduce(wire, dist.ReduceOp.SUM, 1.0), buf)

        def decompress(_f):
            buf.copy_(wire)
            return buf

        return fut.then(decompress)

    return hook


fp16_compress_hook = _compress_hook(torch.float16)
bf16_compress_hook = _compress_hook(torch.bfloat16)


def noop_hook(state, bucket) -> Future:
    """Skips communication (for measuring pure compute); gradients stay local."""
    return Future(None, bucket.buffer())


def fp16_compress_wrapper(hook):
    def wrapped(state, bucket):
        buf = bucket.buffer()
        half = buf.to(torch.float16)
        bucket.set_buffer(half)
        fut = hook(state, bucket)

        def back(f):
            buf.copy_(f._value if isinstance(f, Future) else f)
            return buf

        return fut.then(back)

    return wrapped


class PostLocalSGDState:
    """State for :func:`post_localSGD_hook`: global allreduce for the first ``start_localSGD_iter``
    iterations, then no gradient communication (parameters are averaged periodically by the user)."""

    def __init__(self, process_group=None, start_localSGD_iter: int = 100):
        self.process_group = process_group
        self.start_localSGD_iter = start_localSGD_iter
        self.iter = 0

    def maybe_increase_iter(self, bucket):
        if bucket.is_last():
            self.iter += 1


def post_localSGD_hook(state: PostLocalSGDState, bucket) -> Future:
    if state.iter < state.start_localSGD_iter:
        fut = allreduce_hook(state.process_group, bucket)
    else:
        fut = noop_hook(None, bucket)
    state.maybe_increase_iter(bucket)
    return fut


class PowerSGDState:
    """State for :func:`powerSGD_hook` (rank-r gradient compression with error feedback; the substrate ships the
    same algorithm in ddp_comm_hooks/powerSGD_hook.py — optional surface, unused by the reference).

    For every ≥2-D gradient M (viewed as n×m) the hook communicates P = M·Q (n×r) and Q = Mᵀ·P̂ (m×r) instead of
    M: two small allreduces per bucket.  The compression error is kept per parameter and added back next step.
    1-D tensors, and matrices where r·(n+m) would not save at least ``min_compression_rate``×, travel uncompressed
    in one flat allreduce."""

    def __init__(self, process_group=None, matrix_approximation_rank: int = 1, start_powerSGD_iter: int = 2,
                 min_compression_rate: float = 2.0, use_error_feedback: bool = True, warm_start: bool = True, random_seed: int = 0):
        self.process_group = process_group
        self.rank = int(matrix_approximation_rank)
        self.start_powerSGD_iter = int(start_powerSGD_iter)
        self.min_compression_rate = float(min_compression_rate)
        self.use_error_feedback = use_error_feedback
        self.warm_start = warm_start
        self.rng = torch.Generator().manual_seed(random_seed)   # identical Q on every rank
        self.iter = 0
        self.errors = {}   # (bucket index, slot) -> residual tensor
        self.qs = {}       # (bucket index, slot) -> Q reused across steps (warm start)


def _orthogonalize(p: torch.Tensor) -> torch.Tensor:
    q, _ = torch.linalg.qr(p.float(), mode="reduced")
    return q.to(p.dtype)


def powerSGD_hook(state: PowerSGDState, bucket) -> Future:
    g = _group(state.process_group)
    world = g.size()
    if state.iter < state.start_powerSGD_iter:
        fut = allreduce_hook(g, bucket)
        if bucket.is_last():
            state.iter += 1
        return fut
    buf = bucket.buffer()
    grads = bucket.gradients()
    bidx = bucket.index()
    plain, low = [], []
    for slot, t in enumerate(grads):
        n = t.shape[0] if t.dim() >= 2 else 0
        m = t.numel() // n if n else 0
        r = min(state.rank, n, m) if n else 0
        if n and r * (n + m) * state.min_compression_rate <= n * m:
            low.append((slot, t, n, m, r))
        else:
            plain.append(t)
    # uncompressed part: one flat allreduce (mean)
    if plain:
        flat = torch.cat([t.reshape(-1) for t in plain])
        g.comm.allreduce(flat, dist.ReduceOp.SUM, 1.0 / world).wait()
        off = 0
        for t in plain:
            t.copy_(flat[off:off + t.numel()].view_as(t))
            off += t.numel()
    if low:
        mats, ps = [], []
        for slot, t, n, m, r in low:
            M = t.reshape(n, m)
            key = (bidx, slot)
            if state.use_error_feedback and key in state.errors:
                M.add_(state.errors[key])
            q = state.qs.get(key) if state.warm_start else None
            if q is None or q.shape != (m, r):
                q = torch.randn(m, r, generator=state.rng).to(device=M.device, dtype=M.dtype)
                q = _orthogonalize(q)
            mats.append((key, M, q, r))
            ps.append(M @ q)
        flat_p = torch.cat([p.reshape(-1) for p in ps])
        g.comm.allreduce(flat_p, dist.ReduceOp.SUM, 1.0 / world).wait()
        qs, off = [], 0
        for (key, M, q, r), p in zip(mats, ps):
            p_hat = _orthogonalize(flat_p[off:off + p.numel()].view_as(p))
            off += p.numel()
            ps[len(qs)] = p_hat
            qs.append(M.t() @ p_hat)
        flat_q = torch.cat([q.reshape(-1) for q in qs])
        g.comm.allreduce(flat_q, dist.ReduceOp.SUM, 1.0 / world).wait()
        off = 0
        for (key, M, _, r), p_hat, q in zip(mats, ps, qs):
            q_avg = flat_q[off:off + q.numel()].view_as(q)
            off += q.numel()
            approx = p_hat @ q_avg.t()
            if state.use_error_feedback:
                state.errors[key] = M - approx
            if state.warm_start:
                state.qs[key] = q_avg.clone()
            M.copy_(approx)
    if bucket.is_last():
        state.iter += 1
    return Future(None, buf)
