"""pdt.data.RandomAffine on the native kernel (csrc/cuda/augment.cu): geometry against the float64 reference of
test_random_affine_cpu.py (and torchvision when it is importable) at its tolerances, the exact cases, the parameter distributions,
the Philox stream's reproducibility in and out of CUDA graphs, and GraphedTrainStep(augment=...)."""
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
from test_random_affine_cpu import TVF, check_against_reference, check_against_torchvision

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dev():
    return torch.device("cuda", 0)


# ---- geometry against float64 -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("shape", [(100, 1, 28, 28), (7, 3, 32, 48), (0, 1, 28, 28)])
@pytest.mark.parametrize("interpolation", ["nearest", "bilinear"])
@pytest.mark.parametrize("fill", [0.0, 0.5])
def test_kernel_matches_float64_reference(shape, interpolation, fill):
    x = torch.rand(shape, generator=torch.Generator().manual_seed(2)).to(dev())
    torch.manual_seed(17)
    t = pdt.data.RandomAffine(25, (0.15, 0.1), (0.8, 1.2), (-10, 10, -5, 5), interpolation=interpolation, fill=fill, record_params=True)
    for _ in range(3):   # many draws: 3 calls of the batch
        before = _C.kernel_launch_count()
        out = t(x)
        assert _C.kernel_launch_count() - before == (1 if shape[0] else 0)
        torch.cuda.synchronize()
        assert out.shape == x.shape and out.dtype == torch.float32 and out.is_contiguous()
        p = t.last_params
        assert p.shape == (shape[0], 6) and p.is_cuda and p.dtype == torch.float32
        check_against_reference(x, out, p, interpolation == "bilinear", fill)
        if TVF is not None and shape[0]:
            check_against_torchvision(x, out, p, interpolation == "bilinear", fill)


def test_kernel_shear_only_and_large_scales():
    """Shears and scales far from the identity, where many taps leave the image."""
    x = torch.rand(64, 2, 28, 28, generator=torch.Generator().manual_seed(3)).to(dev())
    torch.manual_seed(4)
    for kw in (dict(degrees=0, shear=(-40, 40, -30, 30)), dict(degrees=180, scale=(0.2, 3.0)), dict(degrees=0, translate=(1.0, 1.0))):
        for interpolation in ("nearest", "bilinear"):
            t = pdt.data.RandomAffine(interpolation=interpolation, fill=0.25, record_params=True, **kw)
            out = t(x)
            check_against_reference(x, out, t.last_params, interpolation == "bilinear", 0.25)


# ---- exact cases ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("shape", [(100, 1, 28, 28), (5, 3, 16, 16)])
def test_exact_cases(shape):
    x = torch.rand(shape, generator=torch.Generator().manual_seed(5)).to(dev())
    # torchvision's 90° turns the picture counter-clockwise on screen (x toward -y): rot90 from W towards H
    assert torch.equal(pdt.data.RandomAffine((90, 90))(x), torch.rot90(x, 1, (-1, -2)))
    assert torch.equal(pdt.data.RandomAffine(0)(x), x)
    assert torch.equal(pdt.data.RandomAffine(0, interpolation="bilinear")(x), x)
    H, W = shape[2:]
    t = pdt.data.RandomAffine(0, translate=(0.25, 0.25), fill=0.75, record_params=True)
    out = t(x)
    for b in range(shape[0]):
        tx, ty = int(t.last_params[b, 1]), int(t.last_params[b, 2])
        ref = torch.full_like(x[b], 0.75)
        ref[:, max(ty, 0):H + min(ty, 0), max(tx, 0):W + min(tx, 0)] = x[b][:, max(-ty, 0):H + min(-ty, 0), max(-tx, 0):W + min(-tx, 0)]
        assert torch.equal(out[b], ref), (b, tx, ty)


def test_dtype_and_generator_checks():
    t = pdt.data.RandomAffine(10)
    for dt in (torch.float64, torch.float16, torch.bfloat16):
        with pytest.raises(TypeError):
            t(torch.zeros(2, 1, 4, 4, dtype=dt, device=dev()))
    with pytest.raises(RuntimeError):
        pdt.data.RandomAffine(10, generator=torch.Generator())(torch.zeros(2, 1, 4, 4, device=dev()))
    # a non-contiguous batch is made contiguous first
    x = torch.rand(8, 8, 1, 6, device=dev()).permute(2, 3, 0, 1)
    torch.manual_seed(1)
    a = pdt.data.RandomAffine(30)(x)
    torch.manual_seed(1)
    assert torch.equal(a, pdt.data.RandomAffine(30)(x.contiguous()))


# ---- distributions ----------------------------------------------------------------------------------------------------------

def test_parameter_distributions():
    from scipy import stats

    x = torch.zeros(4096, 1, 28, 28, device=dev())
    torch.manual_seed(1234)
    t = pdt.data.RandomAffine((-20, 30), (0.1, 0.2), (0.5, 2.0), (1, 2, 3, 4), record_params=True)
    calls = []
    for _ in range(4):
        t(x)
        calls.append(t.last_params.cpu().double())
    for a, b in zip(calls, calls[1:]):
        assert not (a == b).all(1).any()   # consecutive calls draw different parameters
    for c in calls:
        assert len(set(c[:, 0].tolist())) > 4000 and len(set(c[:, 3].tolist())) > 4000   # images within a call differ
    p = torch.cat(calls).numpy()
    for col, lo, hi in ((0, -20, 30), (3, 0.5, 2.0), (4, 1, 2), (5, 3, 4)):
        v = p[:, col]
        assert v.min() >= lo and v.max() < hi, col
        assert stats.kstest(v, stats.uniform(loc=lo, scale=hi - lo).cdf).pvalue > 1e-3, col
    # tx = rint(U[-m, m)): P(k) = |[-m, m) ∩ [k − ½, k + ½]| / 2m (ties to even have measure 0); ty likewise
    for col, m in ((1, 0.1 * 28), (2, 0.2 * 28)):
        v = p[:, col]
        assert (v == np.round(v)).all()
        ks = np.arange(-math.ceil(m), math.ceil(m) + 1)
        prob = np.array([max(0.0, min(m, k + 0.5) - max(-m, k - 0.5)) / (2 * m) for k in ks])
        obs = np.array([(v == k).sum() for k in ks])
        assert obs.sum() == len(v)
        keep = prob > 0
        assert stats.chisquare(obs[keep], prob[keep] * len(v)).pvalue > 1e-3, (col, obs, prob * len(v))


# ---- reproducibility and graphs ---------------------------------------------------------------------------------------------

def _aug(**kw):
    return pdt.data.RandomAffine(20, (0.1, 0.1), (0.9, 1.1), 5, interpolation="bilinear", record_params=True, **kw)


@pytest.mark.parametrize("own_generator", [False, True])
def test_graph_replays_draw_and_reseed(own_generator):
    x = torch.rand(64, 1, 28, 28, generator=torch.Generator().manual_seed(6)).to(dev())
    gen = torch.Generator(device=dev()) if own_generator else None
    seed = (lambda s: gen.manual_seed(s)) if own_generator else torch.manual_seed
    t = _aug(generator=gen)
    seed(5)
    e1, p1 = t(x).clone(), t.last_params.clone()
    e2, p2 = t(x).clone(), t.last_params.clone()
    seed(5)
    assert torch.equal(t(x), e1) and torch.equal(t.last_params, p1)   # the same seed, the same output bit for bit
    g = torch.cuda.CUDAGraph()
    if own_generator:
        g.register_generator_state(gen)
    with torch.cuda.graph(g):
        out = t(x)
    params = t.last_params
    seed(5)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, e1) and torch.equal(params, p1)   # a replay draws what the eager call drew from the same seed
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, e2) and torch.equal(params, p2)   # consecutive replays draw new values, as consecutive calls do
    assert not (p1 == p2).all(1).any()
    seed(5)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, e1)                              # reseeding between replays reproduces the sequence


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


def _step(augment, k=1, seed=0):
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    torch.manual_seed(seed)
    model = pdt.models.ConvNet().to(dev())
    opt = pdt.optim.SGD(model.parameters(), 0.05, momentum=0.9)
    xs = _batches(1, 100 * k)
    step = GraphedTrainStep(pdt.DistributedDataParallel(model, device_ids=[0]), pdt.nn.CrossEntropyLoss(), opt, xs[0], warmup=2,
                            accumulation_steps=k, augment=augment)
    opt.stop_riding()   # the captured graph keeps its rider; the next step captures on its own
    return model, step


def test_identity_augmentation_changes_nothing():
    with _one_gpu():
        xs = _batches(3, 100)
        plain_model, plain = _step(None)
        aug_model, aug = _step(pdt.data.RandomAffine(0))
        assert plain.kernels_per_replay == 3 and aug.kernels_per_replay == plain.kernels_per_replay + 1, (plain.kernels_per_replay,
                                                                                                          aug.kernels_per_replay)
        for r in range(6):
            la, lb = plain(*xs[r % 3]), aug(*xs[r % 3])
            torch.cuda.synchronize()
            assert torch.equal(la, lb), (r, la.item(), lb.item())
        for (n, p), q in zip(plain_model.named_parameters(), aug_model.parameters()):
            assert torch.equal(p, q), n
        for b, c in zip(plain_model.buffers(), aug_model.buffers()):
            assert torch.equal(b, c)


def test_translate_only_step_matches_forward_of_rebuilt_batch():
    with _one_gpu():
        xs = _batches(3, 100)
        t = pdt.data.RandomAffine(0, translate=(0.15, 0.15), record_params=True, generator=torch.Generator(device=dev()))
        model, step = _step(t)
        assert step.kernels_per_replay == 4
        t.generator.manual_seed(3)
        seen = []
        for r in range(6):
            ref = pdt.models.ConvNet().to(dev())
            ref.load_state_dict(model.state_dict())   # the model before this step's update
            x, y = xs[r % 3]
            loss = step(x, y)
            torch.cuda.synchronize()
            p = t.last_params.cpu()
            seen.append(p.clone())
            rebuilt = torch.zeros_like(x)
            for b in range(x.shape[0]):
                tx, ty = int(p[b, 1]), int(p[b, 2])
                rebuilt[b, :, max(ty, 0):28 + min(ty, 0), max(tx, 0):28 + min(tx, 0)] = x[b, :, max(-ty, 0):28 + min(-ty, 0), max(-tx, 0):28 + min(-tx, 0)]
            with torch.no_grad():
                expect = F.cross_entropy(ref(rebuilt).double(), y)
            assert abs(loss.item() - expect.item()) <= 1e-4 * abs(expect.item()), (r, loss.item(), expect.item())
        assert not any(torch.equal(a, b) for a, b in zip(seen, seen[1:]))   # every replay draws new shifts
        # reseeding the registered generator reproduces the first replay's draws
        t.generator.manual_seed(3)
        step(*xs[0])
        torch.cuda.synchronize()
        assert torch.equal(t.last_params.cpu(), seen[0])


def test_accumulation_augments_all_rows_once():
    with _one_gpu():
        t = pdt.data.RandomAffine(10, (0.1, 0.1), record_params=True)
        model, step = _step(t, k=2)
        assert step.kernels_per_replay == 3 * 2 + 1, step.kernels_per_replay
        xs = _batches(2, 200)
        for r in range(4):
            loss = step(*xs[r % 2])
            torch.cuda.synchronize()
            assert math.isfinite(loss.item())
            assert t.last_params.shape == (200, 6)
            assert len(set(t.last_params[:, 0].tolist())) > 190


def test_train_script_with_affine_in_graphed_step():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "1", "--graph", "--rotate", "10", "--translate", "0.1",
                          "--scale-range", "0.9", "1.1", "--steps", "20", "--samples", "4000", "--epochs", "1", "--log-interval", "5",
                          "--eval"],
                         capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    losses = [float(v) for v in re.findall(r"Step \[\d+/\d+\], Loss: (\S+)", out.stdout)]
    assert len(losses) == 4 and all(math.isfinite(v) for v in losses), out.stdout[-1000:]
    assert re.search(r"Test Loss: \S+, Accuracy: \S+% \(10000 images\)", out.stdout), out.stdout[-1000:]
