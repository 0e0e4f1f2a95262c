"""Programmatic dependent launch of the fused ConvNet's backward kernels: the captured training step keeps a programmatic edge
from the forward to the layer-2 backward and from there to the layer-1 backward, so each grid is set up while the kernel
before it finishes.  Behind any other node (an ATen glue kernel, a memset) the capture would record a full dependency instead."""
import contextlib
import functools

import pytest
import torch

import pytorch_distributed_train_b200 as pdt
from pytorch_distributed_train_b200 import _C


def _dev():
    return torch.device("cuda", 0)


@contextlib.contextmanager
def _one_gpu():
    from mp_helpers import free_port

    torch.cuda.set_device(0)
    pdt.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{free_port()}", world_size=1, rank=0)
    try:
        yield
    finally:
        pdt.destroy_process_group()


def _batch(rows, seed):
    g = torch.Generator(device=_dev()).manual_seed(seed)
    return torch.rand(rows, 1, 28, 28, device=_dev(), generator=g), torch.randint(0, 10, (rows,), device=_dev(), generator=g)


def _graphed(monkeypatch, x, t, **kw):
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    # graphs that keep their cudaGraph_t after capture, so that its edges can be read (instantiated on the first replay)
    monkeypatch.setattr(torch.cuda, "CUDAGraph", functools.partial(torch.cuda.CUDAGraph, keep_graph=True))
    torch.manual_seed(0)
    model = pdt.models.ConvNet().to(_dev())
    opt = pdt.optim.SGD(model.parameters(), 0.05, momentum=0.9)
    step = GraphedTrainStep(pdt.DistributedDataParallel(model, device_ids=[0]), pdt.nn.CrossEntropyLoss(), opt, (x, t), warmup=2, **kw)
    monkeypatch.undo()
    return model, step


@pytest.mark.gpu
def test_graphed_step_has_two_programmatic_edges(monkeypatch):
    with _one_gpu():
        x, t = _batch(100, 0)
        model, step = _graphed(monkeypatch, x, t)
        assert step.kernels_per_replay == 3, step.kernels_per_replay
        edges = [_C.graph_programmatic_edges(g.raw_cuda_graph()) for g in step.graphs]
        assert edges == [2] * len(step.graphs), edges   # forward → layer-2 backward → layer-1 backward, in every captured graph
        losses = []
        for i in range(6):
            losses.append(step(*_batch(100, 1 + i % 2)).item())
        torch.cuda.synchronize()
        assert all(torch.isfinite(p).all() for p in model.parameters())
        assert losses[-1] < losses[0], losses


@pytest.mark.gpu
def test_graphed_accumulation_with_clipping_keeps_programmatic_edges(monkeypatch):
    k = 2
    with _one_gpu():
        x, t = _batch(100 * k, 3)
        model, step = _graphed(monkeypatch, x, t, accumulation_steps=k, max_grad_norm=0.5)
        assert step.accumulates_in_kernel and step.kernels_per_replay == 3 * k, step.kernels_per_replay
        edges = [_C.graph_programmatic_edges(g.raw_cuda_graph()) for g in step.graphs]
        assert edges == [2 * k] * len(step.graphs), edges
        norms = []
        for i in range(4):
            step(*_batch(100 * k, 4 + i % 2))
            norms.append(step.grad_norm.item())
        torch.cuda.synchronize()
        assert all(n > 0 and n == n for n in norms), norms
        assert all(torch.isfinite(p).all() for p in model.parameters())
