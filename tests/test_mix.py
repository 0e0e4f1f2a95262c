"""pdt.data.MixUp and pdt.data.CutMix on the native kernel (csrc/cuda/augment.cu, mix_batch_kernel): images and targets bit for bit
against the float64 reference of test_mix_cpu.py given the recorded parameters, the distributions of λ, r_x and r_y, the Philox
stream's reproducibility in and out of CUDA graphs, and GraphedTrainStep(mix=...)."""
import contextlib
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import pytorch_distributed_train_b200 as pdt
from pytorch_distributed_train_b200 import _C
from test_mix_cpu import check_against_reference, cutmix_box, reference_mix

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dev():
    return torch.device("cuda", 0)


def _labels(B, prob, seed=0, K=10):
    g = torch.Generator().manual_seed(seed)
    y = torch.softmax(torch.randn(B, K, generator=g), 1) if prob else torch.randint(0, K, (B,), generator=g)
    return y.to(dev())


def _mix(cutmix, **kw):
    return (pdt.data.CutMix if cutmix else pdt.data.MixUp)(**kw)


# ---- outputs against float64 ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cutmix", [False, True])
@pytest.mark.parametrize("shape", [(100, 1, 28, 28), (7, 3, 16, 20), (1, 1, 28, 28), (0, 1, 28, 28)])
@pytest.mark.parametrize("prob", [False, True])
def test_kernel_matches_float64_reference(cutmix, shape, prob):
    x = torch.rand(shape, generator=torch.Generator().manual_seed(2)).to(dev())
    y = _labels(shape[0], prob, seed=3)
    torch.manual_seed(11)
    t = _mix(cutmix, alpha=0.7, num_classes=10, record_params=True)
    for _ in range(8):
        before = _C.kernel_launch_count()
        out, targets = t(x, y)
        assert _C.kernel_launch_count() - before == (1 if shape[0] else 0)
        torch.cuda.synchronize()
        assert out.shape == x.shape and out.dtype == torch.float32 and out.is_cuda and out.is_contiguous()
        assert targets.shape == (shape[0], 10) and targets.dtype == torch.float32 and targets.is_cuda
        rec = t.last_params
        assert rec.dtype == torch.float64 and rec.is_cuda and rec.shape == ((8,) if cutmix else (1,))
        if shape[0]:
            check_against_reference(x, y, 10, out, targets, rec, cutmix)
        else:
            assert torch.isnan(rec).all()   # nothing drawn


@pytest.mark.parametrize("cutmix", [False, True])
def test_out_of_range_labels_add_no_mass(cutmix):
    x = torch.rand(6, 1, 8, 8, device=dev())
    y = torch.tensor([0, -1, 10, 3, 12345, 9], device=dev())
    t = _mix(cutmix, alpha=1.0, num_classes=10, record_params=True)
    out, targets = t(x, y)
    torch.cuda.synchronize()
    check_against_reference(x, y, 10, out, targets, t.last_params, cutmix)
    lam = float(t.last_params[-1 if cutmix else 0])
    # row 2 pairs label 10 with label -1: no mass at all; row 1 keeps only its partner's share
    assert float(targets[2].sum()) == 0.0
    assert float(targets[1, 0]) == np.float32(1.0 - lam)


def test_non_contiguous_and_device_checks():
    x = torch.rand(8, 8, 1, 6, device=dev()).permute(2, 3, 0, 1)   # [1, 6, 8, 8], not contiguous
    y = torch.randint(0, 10, (1,), device=dev())
    torch.manual_seed(1)
    a, ta = pdt.data.CutMix(num_classes=10)(x, y)
    torch.manual_seed(1)
    b, tb = pdt.data.CutMix(num_classes=10)(x.contiguous(), y)
    assert torch.equal(a, b) and torch.equal(ta, tb)
    with pytest.raises(ValueError):
        pdt.data.MixUp(num_classes=10)(x.contiguous(), y.cpu())
    with pytest.raises(RuntimeError):
        pdt.data.MixUp(num_classes=10, generator=torch.Generator())(x.contiguous(), y)


# ---- distributions ----------------------------------------------------------------------------------------------------------

def _records(t, x, y, n):
    recs = []
    for _ in range(n):
        t(x, y)
        recs.append(t.last_params)
    return torch.stack(recs).cpu().numpy()


@pytest.mark.parametrize("alpha", [0.1, 0.2, 1.0, 5.0])
def test_lambda_is_beta(alpha):
    from scipy import stats

    torch.manual_seed(100 + int(10 * alpha))
    x, y = torch.rand(2, 1, 4, 4, device=dev()), torch.randint(0, 10, (2,), device=dev())
    lam = _records(pdt.data.MixUp(alpha=alpha, num_classes=10, record_params=True), x, y, 4000)[:, 0]
    assert np.isfinite(lam).all() and lam.min() >= 0.0 and lam.max() <= 1.0
    assert stats.kstest(lam, stats.beta(alpha, alpha).cdf).pvalue > 1e-3
    # no repeats: at α = 0.1 about 1% of the draws round to exactly 0 or 1 in double (1 − λ < 2⁻⁵³), so only the interior is unique
    inner = lam[(lam > 1e-9) & (lam < 1 - 1e-9)]
    assert len(inner) > 0.5 * len(lam) and len(np.unique(inner)) == len(inner)
    assert abs(np.corrcoef(lam[:-1], lam[1:])[0, 1]) < 4 / math.sqrt(len(lam))   # no lag-1 correlation


def test_tiny_alpha_stays_finite():
    torch.manual_seed(5)
    x, y = torch.rand(3, 1, 4, 4, device=dev()), torch.randint(0, 10, (3,), device=dev())
    t = pdt.data.CutMix(alpha=0.01, num_classes=10, record_params=True)
    rec = _records(t, x, y, 2000)
    assert np.isfinite(rec).all() and rec[:, 0].min() >= 0.0 and rec[:, 0].max() <= 1.0
    assert ((rec[:, 0] < 1e-3) | (rec[:, 0] > 1 - 1e-3)).mean() > 0.85   # Beta(0.01, 0.01) puts about 93% there
    out, targets = t(x, y)
    assert torch.isfinite(out).all() and torch.isfinite(targets).all()


def test_box_draws_are_uniform_and_follow_torchvision():
    from scipy import stats

    torch.manual_seed(6)
    H, W = 16, 20
    x, y = torch.rand(2, 1, H, W, device=dev()), torch.randint(0, 10, (2,), device=dev())
    rec = _records(pdt.data.CutMix(alpha=1.0, num_classes=10, record_params=True), x, y, 4000)
    for col, n in ((1, W), (2, H)):
        v = rec[:, col]
        assert (v == np.round(v)).all() and v.min() >= 0 and v.max() <= n - 1
        obs = np.bincount(v.astype(np.int64), minlength=n)
        assert stats.chisquare(obs).pvalue > 1e-3, (col, obs)
    for r in rec:
        box, lam_adj = cutmix_box(r[0], r[1], r[2], H, W)
        assert box == tuple(int(v) for v in r[3:7]) and lam_adj == r[7], r
    assert stats.kstest(rec[:, 0], stats.beta(1.0, 1.0).cdf).pvalue > 1e-3


# ---- reproducibility and graphs ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cutmix", [False, True])
@pytest.mark.parametrize("own_generator", [False, True])
def test_graph_replays_draw_and_reseed(cutmix, own_generator):
    x = torch.rand(64, 1, 28, 28, generator=torch.Generator().manual_seed(6)).to(dev())
    y = _labels(64, False, seed=7)
    gen = torch.Generator(device=dev()) if own_generator else None
    seed = (lambda s: gen.manual_seed(s)) if own_generator else torch.manual_seed
    t = _mix(cutmix, alpha=1.0, num_classes=10, generator=gen, record_params=True)
    seed(5)
    e1, q1, p1 = (v.clone() for v in (*t(x, y), t.last_params))
    e2, q2, p2 = (v.clone() for v in (*t(x, y), t.last_params))
    assert not torch.equal(p1, p2)
    seed(5)
    out, q = t(x, y)
    assert torch.equal(out, e1) and torch.equal(q, q1) and torch.equal(t.last_params, p1)   # the same seed, the same output
    g = torch.cuda.CUDAGraph()
    if own_generator:
        g.register_generator_state(gen)
    with torch.cuda.graph(g):
        out, q = t(x, y)
    params = t.last_params
    seed(5)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, e1) and torch.equal(q, q1) and torch.equal(params, p1)   # a replay draws what the eager call drew
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, e2) and torch.equal(params, p2)   # consecutive replays draw anew, as consecutive calls do
    seed(5)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(params, p1)                            # reseeding between replays reproduces the sequence


# ---- the graphed training step ----------------------------------------------------------------------------------------------

@contextlib.contextmanager
def _one_gpu():
    from mp_helpers import free_port

    torch.cuda.set_device(0)
    pdt.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{free_port()}", world_size=1, rank=0)
    try:
        yield
    finally:
        pdt.destroy_process_group()


def _batches(n, rows):
    out = []
    for i in range(n):
        gen = torch.Generator().manual_seed(60 + i)
        out.append((torch.rand(rows, 1, 28, 28, generator=gen).to(dev()), torch.randint(0, 10, (rows,), generator=gen).to(dev())))
    return out


def _step(mix=None, augment=None, k=1, seed=0):
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    torch.manual_seed(seed)
    model = pdt.models.ConvNet().to(dev())
    opt = pdt.optim.SGD(model.parameters(), 0.05, momentum=0.9)
    step = GraphedTrainStep(pdt.DistributedDataParallel(model, device_ids=[0]), pdt.nn.CrossEntropyLoss(), opt, _batches(1, 100 * k)[0],
                            warmup=2, accumulation_steps=k, augment=augment, mix=mix)
    opt.stop_riding()   # the captured graph keeps its rider; the next step captures on its own
    return model, step


def _expected_loss(model_before, x, y, record, k):
    """The step's loss from a copy of the pre-step model on the batch and targets rebuilt from the record: the mean of the k
    micro-batches' mean cross-entropies (BatchNorm statistics per micro-batch)."""
    mx, mt = reference_mix(x, y, 10, record, True)
    mx, mt = mx.to(dev()), mt.to(dev())
    b = x.shape[0] // k
    with torch.no_grad():
        parts = [F.cross_entropy(model_before(mx[i * b:(i + 1) * b]).double(), mt[i * b:(i + 1) * b].double()) for i in range(k)]
    return float(sum(parts) / k)


@pytest.mark.parametrize("k", [1, 2])
def test_graphed_step_with_cutmix_matches_rebuilt_batch(k):
    with _one_gpu():
        xs = _batches(3, 100 * k)
        _, plain = _step(k=k)
        t = pdt.data.CutMix(alpha=1.0, num_classes=10, record_params=True, generator=torch.Generator(device=dev()))
        model, step = _step(mix=t, k=k)
        assert step.kernels_per_replay == plain.kernels_per_replay + 1, (plain.kernels_per_replay, step.kernels_per_replay)
        if k == 2:
            assert step.kernels_per_replay == 7
        t.generator.manual_seed(3)
        seen = []
        for r in range(6):
            ref = pdt.models.ConvNet().to(dev())
            ref.load_state_dict(model.state_dict())   # the model before this step's update
            x, y = xs[r % 3]
            loss = step(x, y)
            torch.cuda.synchronize()
            rec = t.last_params.cpu()
            seen.append(rec.clone())
            expect = _expected_loss(ref, x, y, rec, k)
            assert abs(loss.item() - expect) <= 1e-4 * abs(expect), (r, loss.item(), expect)
        assert not any(torch.equal(a, b) for a, b in zip(seen, seen[1:]))   # every replay draws a new box
        t.generator.manual_seed(3)
        step(*xs[0])
        torch.cuda.synchronize()
        assert torch.equal(t.last_params.cpu(), seen[0])   # reseeding the registered generator reproduces the first replay's draws


def test_graphed_step_with_affine_and_cutmix():
    with _one_gpu():
        _, plain = _step()
        aff = pdt.data.RandomAffine(10, (0.1, 0.1), record_params=True, generator=torch.Generator(device=dev()))
        cut = pdt.data.CutMix(alpha=1.0, num_classes=10, record_params=True, generator=torch.Generator(device=dev()))
        _, step = _step(mix=cut, augment=aff)
        assert step.kernels_per_replay == plain.kernels_per_replay + 2
        xs = _batches(2, 100)
        recs = []
        for r in range(4):
            loss = step(*xs[r % 2])
            torch.cuda.synchronize()
            assert math.isfinite(loss.item())
            recs.append((aff.last_params.clone(), cut.last_params.clone()))
        for (a0, c0), (a1, c1) in zip(recs, recs[1:]):
            assert not torch.equal(a0, a1) and not torch.equal(c0, c1)   # both transforms draw anew on every replay


def test_train_script_with_cutmix_in_graphed_step():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "1", "--graph", "--cutmix", "1.0", "--rotate", "10",
                          "--steps", "20", "--samples", "4000", "--epochs", "1", "--log-interval", "5", "--eval"],
                         capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    losses = [float(v) for v in re.findall(r"Step \[\d+/\d+\], Loss: (\S+)", out.stdout)]
    assert len(losses) == 4 and all(math.isfinite(v) for v in losses), out.stdout[-1000:]
    assert re.search(r"Test Loss: \S+, Accuracy: \S+% \(10000 images\)", out.stdout), out.stdout[-1000:]
