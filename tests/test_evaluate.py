"""Test-set evaluation (engine.evaluate) and the cross-entropy kernel's accumulate mode (_C.cross_entropy_eval).

CPU: evaluate on the gloo backend at world sizes 1-4 over a split that no world size divides, against F.cross_entropy over the
concatenated float64 logits; the model's state and mode untouched; the CLI's --eval lines.  GPU: the kernel against a float64 oracle,
evaluate against the same eval forward's logits, no host synchronisation in the batch loop, one launch per batch on top of the
forward, and a graphed training run that an evaluation in the middle does not change."""
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import pytorch_distributed_train_b200 as pdt
from mp_helpers import run_ranks
from pytorch_distributed_train_b200.data import DataLoader, DistributedSampler, SyntheticMNIST, TensorDataset
from pytorch_distributed_train_b200.optim import swa_utils

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

N_SPLIT, BATCH, IGNORE = 1001, 64, 3


# ---- CPU: the torch-op path, exact across ranks --------------------------------------------------------------------------------
def _split():
    x, y = SyntheticMNIST(N_SPLIT, seed=1).gather(list(range(N_SPLIT)))
    y_ignored = y.clone()
    y_ignored[::7] = IGNORE   # ignored: every 7th row and every row of that class
    return x, y, y_ignored


def _cpu_model():
    torch.manual_seed(0)
    return nn.Sequential(nn.Flatten(), nn.Linear(784, 10))


def _cases():
    w = torch.rand(10, generator=torch.Generator().manual_seed(4)) + 0.25
    return {
        "plain": dict(),
        "shuffle": dict(shuffle=True),
        "drop_last": dict(drop_last=True),
        "weight": dict(criterion=pdt.nn.CrossEntropyLoss(weight=w)),
        "smoothing": dict(criterion=nn.CrossEntropyLoss(label_smoothing=0.1)),   # torch's criterion is accepted too
        "ignore_index": dict(criterion=pdt.nn.CrossEntropyLoss(ignore_index=IGNORE), ignored=True),
        "sum": dict(criterion=pdt.nn.CrossEntropyLoss(weight=w, reduction="sum", label_smoothing=0.2)),
        "ddp": dict(ddp=True),
    }


def _evaluate_rank(rank, world):
    x, y, y_ignored = _split()
    out = {}
    for name, c in _cases().items():
        ds = TensorDataset(x, y_ignored if c.get("ignored") else y)
        sampler = DistributedSampler(ds, world, rank, shuffle=c.get("shuffle", False), seed=11, drop_last=c.get("drop_last", False))
        model = _cpu_model()
        if c.get("ddp"):
            model = pdt.DistributedDataParallel(model)
        out[name] = (pdt.engine.evaluate(model, DataLoader(ds, batch_size=BATCH, sampler=sampler), c.get("criterion")),
                     sorted(sampler))
    return out


def _oracle(name, c, indices):
    """loss and correct of the criterion over the concatenated float64 logits of the split's images at ``indices``."""
    x, y, y_ignored = _split()
    t = (y_ignored if c.get("ignored") else y)[indices]
    with torch.no_grad():
        logits = _cpu_model()(x[indices]).double()
    crit = c.get("criterion") or pdt.nn.CrossEntropyLoss()
    w = None if crit.weight is None else crit.weight.double()
    loss = F.cross_entropy(logits, t, w, ignore_index=crit.ignore_index, reduction=crit.reduction, label_smoothing=crit.label_smoothing)
    counted = t != crit.ignore_index
    return loss.item(), int(((logits.argmax(1) == t) & counted).sum()), int(counted.sum())


def test_evaluate_gloo_counts_every_image_once_at_any_world_size():
    results = {world: run_ranks(_evaluate_rank, world) for world in (1, 2, 3, 4)}
    for name, c in _cases().items():
        for world, per_rank in results.items():
            res = [r[name][0] for r in per_rank]
            assert all(r == res[0] for r in res), (name, world, res)   # every rank returns the all-reduced totals
            got = res[0]
            if c.get("drop_last"):
                indices = sorted(i for r in per_rank for i in r[name][1])   # what the sampler yields: the tail is dropped
                assert len(indices) == world * (N_SPLIT // world)
            else:
                indices = list(range(N_SPLIT))
            loss, correct, count = _oracle(name, c, torch.tensor(indices))
            assert got["count"] == count, (name, world, got)
            assert got["correct"] == correct, (name, world, got, correct)
            if not c.get("drop_last"):   # the same images as in one process: the same count
                assert got["correct"] == results[1][0][name][0]["correct"], (name, world)
            assert abs(got["loss"] - loss) <= 1e-6 * abs(loss), (name, world, got["loss"], loss)
            assert got["accuracy"] == correct / count
    assert results[1][0]["plain"][0]["count"] == N_SPLIT


def test_evaluate_leaves_the_model_as_it_was():
    torch.manual_seed(0)
    model = pdt.models.ConvNet()
    before = {k: v.clone() for k, v in model.state_dict().items()}
    x, y, _ = _split()
    loader = DataLoader(TensorDataset(x[:300], y[:300]), batch_size=BATCH)
    for mode in (True, False):
        model.train(mode)
        r = pdt.engine.evaluate(model, loader)
        assert model.training is mode and r["count"] == 300
        for k, v in model.state_dict().items():
            assert torch.equal(v, before[k]), k
    with pytest.raises(ValueError, match="criterion must be"):
        pdt.engine.evaluate(model, loader, nn.MSELoss())
    with pytest.raises(ValueError, match="reduction"):
        pdt.engine.evaluate(model, loader, pdt.nn.CrossEntropyLoss(reduction="none"))


def _cli(*extra):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "2", "--backend", "gloo", "--epochs", "1",
                          "--steps", "3", "--log-interval", "1", *extra], capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    return out.stdout.splitlines()


def test_cli_eval_prints_the_test_lines_and_nothing_else_changes():
    plain = _cli("--ema-decay", "0.9")
    evaluated = _cli("--ema-decay", "0.9", "--eval")
    test = [l for l in evaluated if "Test Loss" in l]
    assert len(test) == 2, evaluated
    assert test[0].startswith("Epoch [1/1], Test Loss: ") and test[0].endswith("(10000 images)"), test
    assert test[1].startswith("Epoch [1/1], EMA Test Loss: ") and test[1].endswith("(10000 images)"), test
    assert "Accuracy: " in test[0] and "%" in test[0]
    timeless = lambda lines: sorted(l for l in lines if not l.startswith("Training complete in: "))   # noqa: E731
    assert timeless(plain) == timeless(l for l in evaluated if "Test Loss" not in l)
    assert not any("Test Loss" in l for l in plain)


# ---- GPU: the kernel's accumulate mode -----------------------------------------------------------------------------------------
def _dev():
    return torch.device("cuda", torch.cuda.current_device())


def _acc_oracle(x, t, rows, w, ignore_index, eps):
    """acc[0..3] in float64 on the CPU: Σ terms, Σ counted target weights, top-1 hits, counted rows of the first ``rows`` rows."""
    xd, tc = x[:rows].double().cpu(), t[:rows].cpu()
    C = x.shape[1]
    counted = (tc >= 0) & (tc < C) & (tc != ignore_index)
    safe = torch.where(counted, tc, 0)
    wd = None if w is None else w.double().cpu()
    terms = F.cross_entropy(xd, safe, wd, reduction="none", label_smoothing=eps)[counted]
    w_t = torch.ones(int(counted.sum()), dtype=torch.float64) if wd is None else wd[safe[counted]]
    hits = ((x[:rows].cpu().argmax(1) == tc) & counted).sum()
    return terms.sum().item(), w_t.sum().item(), int(hits), int(counted.sum())


@pytest.mark.gpu
@pytest.mark.parametrize("C", [2, 10, 16, 1000])
@pytest.mark.parametrize("B", [1, 7, 100, 300])
def test_cross_entropy_eval_matches_float64(B, C):
    gen = torch.Generator(device=_dev()).manual_seed(B * 31 + C)
    for variant in ("plain", "ties", "nan"):
        x = torch.randn(B, C, device=_dev(), generator=gen)
        t = torch.randint(0, C, (B,), device=_dev(), generator=gen)
        if variant == "ties":   # every row's maximum twice: argmax is the first of them
            x[:, C - 1] = x.max(1).values
            t[::2] = C - 1
        if variant == "nan":
            x[0, C // 2] = float("nan")
            x[0, C - 1] = float("nan")
            t[0] = C // 2
        for wkind in ("none", "random"):
            w = None if wkind == "none" else torch.rand(C, device=_dev(), generator=gen) + 0.25
            for eps in (0.0, 0.1):
                for ignore_index in (-100, 1):
                    tt = t.clone()
                    if B > 2:
                        tt[1::3] = ignore_index
                        tt[2::5] = C + 3     # out of range: not counted, as in the loss
                        tt[3::7] = -5
                    for rows in sorted({B, B // 2, 0}):
                        acc = torch.zeros(4, dtype=torch.float64, device=_dev())
                        pdt._C.cross_entropy_eval(x, tt, acc, rows, w, ignore_index, eps)
                        got = acc.tolist()
                        ref = _acc_oracle(x, tt, rows, w, ignore_index, eps)
                        case = (variant, wkind, eps, ignore_index, rows)
                        assert got[2] == ref[2] and got[3] == ref[3], (case, got, ref)
                        if math.isnan(ref[0]):   # a counted NaN row
                            assert math.isnan(got[0]), (case, got)
                        else:
                            # test_cross_entropy_options.py's tolerance on the mean Σ/D, carried to the sum
                            assert abs(got[0] - ref[0]) <= 1e-5 * abs(ref[0]) + 1e-6 * max(ref[1], 1.0), (case, got, ref)
                        assert abs(got[1] - ref[1]) <= 1e-5 * abs(ref[1]) + 1e-6, (case, got, ref)


@pytest.mark.gpu
def test_cross_entropy_eval_accumulates_bit_reproducibly():
    gen = torch.Generator(device=_dev()).manual_seed(5)
    xs = torch.randn(50, 300, 100, device=_dev(), generator=gen)
    ts = torch.randint(0, 100, (50, 300), device=_dev(), generator=gen)
    w = torch.rand(100, device=_dev(), generator=gen) + 0.25
    runs = []
    for _ in range(3):
        acc = torch.zeros(4, dtype=torch.float64, device=_dev())
        for x, t in zip(xs, ts):
            pdt._C.cross_entropy_eval(x, t, acc, 300, w, -100, 0.1)
        runs.append(acc.clone())
    assert torch.equal(runs[0], runs[1]) and torch.equal(runs[0], runs[2])
    assert runs[0][3].item() == 50 * 300


@pytest.mark.gpu
def test_cross_entropy_eval_rejects_bad_arguments():
    x = torch.randn(8, 10, device=_dev())
    t = torch.randint(0, 10, (8,), device=_dev())
    with pytest.raises(RuntimeError, match="acc"):
        pdt._C.cross_entropy_eval(x, t, torch.zeros(4, device=_dev()), 8)
    with pytest.raises(RuntimeError, match="rows"):
        pdt._C.cross_entropy_eval(x, t, torch.zeros(4, dtype=torch.float64, device=_dev()), 9)
    with pytest.raises(RuntimeError, match="C <= 1024"):
        pdt._C.cross_entropy_eval(torch.randn(8, 1025, device=_dev()), t, torch.zeros(4, dtype=torch.float64, device=_dev()), 8)


# ---- GPU: evaluate on the ConvNet ----------------------------------------------------------------------------------------------
def _trained_convnet(num_classes=10, steps=5):
    torch.manual_seed(0)
    model = pdt.models.ConvNet(num_classes=num_classes).to(_dev())
    opt = pdt.optim.SGD(model.parameters(), 0.05)
    ema = swa_utils.AveragedModel(model, multi_avg_fn=swa_utils.get_ema_multi_avg_fn(0.5), use_buffers=True)
    crit = pdt.nn.CrossEntropyLoss()
    g = torch.Generator(device=_dev()).manual_seed(3)
    for _ in range(steps):
        x = torch.rand(100, 1, 28, 28, device=_dev(), generator=g)
        y = torch.randint(0, num_classes, (100,), device=_dev(), generator=g)
        opt.zero_grad()
        crit(model(x), y).backward()
        opt.step()
        ema.update_parameters(model)
    return model, ema


def _gpu_loader(n=1050, num_classes=10, batch=100):
    ds = SyntheticMNIST(n, seed=1, num_classes=num_classes)
    return DataLoader(ds, batch_size=batch, pin_memory=True)


def _eval_logits(model, loader):
    was = model.training
    model.eval()
    with torch.no_grad():
        pairs = [(model(x.to(_dev())), y.to(_dev())) for x, y in loader]
    model.train(was)
    return torch.cat([p[0] for p in pairs]), torch.cat([p[1] for p in pairs])


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["convnet", "averaged", "classes40"])
def test_evaluate_convnet_matches_its_eval_logits(which):
    model, ema = _trained_convnet(num_classes=40 if which == "classes40" else 10)
    net = ema if which == "averaged" else model
    loader = _gpu_loader(num_classes=40 if which == "classes40" else 10)
    state = {k: v.clone() for k, v in net.state_dict().items()}
    got = pdt.engine.evaluate(net, loader)
    logits, y = _eval_logits(net, loader)
    assert got["count"] == 1050
    assert got["correct"] == int((logits.argmax(1) == y).sum())
    ref = F.cross_entropy(logits.double(), y).item()
    assert abs(got["loss"] - ref) <= 1e-5 * abs(ref) + 1e-6, (got, ref)
    assert net.training
    for k, v in net.state_dict().items():
        assert torch.equal(v, state[k]), k


class _SyncForbidden:
    """A loader whose batches are consumed with torch's synchronisation check set to raise."""

    def __init__(self, loader):
        self.loader, self.sampler = loader, loader.sampler

    def __iter__(self):
        torch.cuda.set_sync_debug_mode("error")
        try:
            yield from self.loader
        finally:
            torch.cuda.set_sync_debug_mode(0)


@pytest.mark.gpu
def test_evaluate_batch_loop_does_not_synchronise_and_adds_one_launch_per_batch():
    model, _ = _trained_convnet()
    loader = _gpu_loader(n=1000)
    ref = pdt.engine.evaluate(model, loader)
    assert pdt.engine.evaluate(model, _SyncForbidden(loader)) == ref
    x = next(iter(loader))[0].to(_dev())
    model.eval()
    with torch.no_grad():
        model(x)
        before = pdt._C.kernel_launch_count()
        model(x)
        forward = pdt._C.kernel_launch_count() - before
    model.train()
    before = pdt._C.kernel_launch_count()
    pdt.engine.evaluate(model, loader)
    assert pdt._C.kernel_launch_count() - before == len(loader) * (forward + 1), forward


def _graphed_training(with_eval):
    from mp_helpers import free_port

    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    torch.cuda.set_device(0)
    pdt.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{free_port()}", world_size=1, rank=0)
    try:
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(_dev())
        ddp = pdt.DistributedDataParallel(model, device_ids=[0])
        g = torch.Generator(device=_dev()).manual_seed(9)
        xs = torch.rand(4, 100, 1, 28, 28, device=_dev(), generator=g)
        ts = torch.randint(0, 10, (4, 100), device=_dev(), generator=g)
        step = GraphedTrainStep(ddp, pdt.nn.CrossEntropyLoss(), pdt.optim.SGD(model.parameters(), 0.05, momentum=0.9), (xs[0], ts[0]))
        losses = [step(xs[i % 4], ts[i % 4], inputs_ready=True).clone() for i in range(4)]
        if with_eval:
            assert pdt.engine.evaluate(ddp, _gpu_loader())["count"] == 1050
        losses += [step(xs[i % 4], ts[i % 4], inputs_ready=True).clone() for i in range(4)]
        torch.cuda.synchronize()
        return torch.stack(losses), {k: v.clone() for k, v in model.state_dict().items()}
    finally:
        pdt.destroy_process_group()


@pytest.mark.gpu
def test_evaluate_between_graph_replays_changes_no_bit_of_training():
    plain_losses, plain_state = _graphed_training(False)
    losses, state = _graphed_training(True)
    assert torch.equal(losses, plain_losses)
    for k, v in state.items():
        assert torch.equal(v, plain_state[k]), k


# ---- two GPUs: DDP on the NVLink backend (skips with fewer than two) -----------------------------------------------------------
def _evaluate_two_gpus(rank, world):
    model, _ = _trained_convnet()
    ddp = pdt.DistributedDataParallel(model, device_ids=[rank])
    ds = SyntheticMNIST(N_SPLIT, seed=1)
    sampler = DistributedSampler(ds, world, rank, shuffle=False)
    loader = DataLoader(ds, batch_size=BATCH, sampler=sampler, pin_memory=True)
    got = pdt.engine.evaluate(ddp, loader)
    logits, y = _eval_logits(model, loader)
    real = len(range(rank, N_SPLIT, world))   # this rank's images before the padding
    return got, logits[:real].cpu(), y[:real].cpu()


@pytest.mark.gpu
@pytest.mark.multigpu
def test_evaluate_ddp_two_gpus():
    res = run_ranks(_evaluate_two_gpus, 2, backend="nccl")
    logits = torch.cat([r[1] for r in res])
    y = torch.cat([r[2] for r in res])
    assert res[0][0] == res[1][0]
    got = res[0][0]
    assert got["count"] == N_SPLIT and logits.shape[0] == N_SPLIT
    assert got["correct"] == int((logits.argmax(1) == y).sum())
    ref = F.cross_entropy(logits.double(), y).item()
    assert abs(got["loss"] - ref) <= 1e-5 * abs(ref) + 1e-6
