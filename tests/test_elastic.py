"""pdt.data.ElasticTransform on the native kernel (csrc/cuda/augment.cu): output against the float64 reference of
test_elastic_cpu.py (and torchvision when it is importable) at its tolerances, the exact cases, the noise's distribution and
independence, the Philox stream's reproducibility in and out of CUDA graphs, GraphedTrainStep(augment=...) with the elastic
transform alone and after RandomAffine, and the graphed CLI."""
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
from test_elastic_cpu import CASES, TVF, check_against_reference, check_against_torchvision, sample, source_coords
from test_random_affine_cpu import reference as affine_reference

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dev():
    return torch.device("cuda", 0)


# ---- output against float64 -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("shape, alpha, sigma", CASES + [((100, 1, 28, 28), 50.0, 5.0), ((64, 1, 32, 32), 50.0, (5.0, 2.0))])
@pytest.mark.parametrize("interpolation", ["nearest", "bilinear"])
@pytest.mark.parametrize("fill", [0.0, 0.5])
def test_kernel_matches_float64_reference(shape, alpha, sigma, interpolation, fill):
    x = torch.rand(shape, generator=torch.Generator().manual_seed(2)).to(dev())
    torch.manual_seed(17)
    t = pdt.data.ElasticTransform(alpha, sigma, interpolation=interpolation, fill=fill, record_params=True)
    for _ in range(2):
        before = _C.kernel_launch_count()
        out = t(x)
        assert _C.kernel_launch_count() - before == (1 if shape[0] else 0)
        torch.cuda.synchronize()
        assert out.shape == x.shape and out.dtype == torch.float32 and out.is_contiguous()
        n = t.last_params
        assert n.shape == (shape[0], 2) + shape[2:] and n.is_cuda and n.dtype == torch.float32
        tol = check_against_reference(x, out, n, t.alpha, t.sigma, interpolation == "bilinear", fill)
        if TVF is not None and shape[0]:
            check_against_torchvision(x, out, n, t.alpha, t.sigma, interpolation == "bilinear", fill, tol)


def test_exact_cases_and_checks():
    x = torch.rand(50, 3, 28, 28, generator=torch.Generator().manual_seed(5)).to(dev())
    for interpolation in ("nearest", "bilinear"):
        for sigma in (5.0, 0.0):
            assert torch.equal(pdt.data.ElasticTransform(0.0, sigma, interpolation=interpolation)(x), x)
    empty = torch.rand(0, 1, 28, 28, device=dev())
    before = _C.kernel_launch_count()
    assert pdt.data.ElasticTransform()(empty).shape == empty.shape and _C.kernel_launch_count() == before
    t = pdt.data.ElasticTransform()
    for dt in (torch.float64, torch.float16, torch.bfloat16):
        with pytest.raises(TypeError):
            t(torch.zeros(2, 1, 28, 28, dtype=dt, device=dev()))
    with pytest.raises(RuntimeError):
        pdt.data.ElasticTransform(generator=torch.Generator())(torch.zeros(2, 1, 28, 28, device=dev()))
    with pytest.raises(RuntimeError, match="Padding size should be less"):
        pdt.data.ElasticTransform(sigma=7.0)(torch.zeros(2, 1, 28, 28, device=dev()))
    # a size whose three fp32 planes exceed the opt-in shared memory is refused, naming the limit
    limit = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    side = int(math.isqrt(limit // 12)) + 1
    with pytest.raises(ValueError, match=f"opt-in limit of {limit} bytes"):
        pdt.data.ElasticTransform(sigma=0.0)(torch.zeros(1, 1, side, side, device=dev()))
    big = torch.rand(2, 1, side - 1, side - 1, device=dev())
    assert torch.equal(pdt.data.ElasticTransform(0.0, 5.0)(big), big)   # the largest square that fits runs natively
    # a non-contiguous batch is made contiguous first
    x = torch.rand(28, 28, 4, 1, device=dev()).permute(2, 3, 0, 1)
    torch.manual_seed(1)
    a = pdt.data.ElasticTransform()(x)
    torch.manual_seed(1)
    assert torch.equal(a, pdt.data.ElasticTransform()(x.contiguous()))


def test_unblurred_displacement_is_exact():
    """sigma <= 0: no blur, the displacement is fl(fl(noise·alpha)/W) bit for bit, so the nearest output is bit-equal everywhere."""
    x = torch.rand(16, 2, 28, 32, generator=torch.Generator().manual_seed(7)).to(dev())
    t = pdt.data.ElasticTransform(37.3, -1.0, interpolation="nearest", fill=0.25, record_params=True)
    out, n = t(x).cpu(), t.last_params.cpu()
    xc = x.cpu()
    for b in range(16):
        dx, dy = (n[b, 0] * 37.3 / 32).double().numpy(), (n[b, 1] * 37.3 / 28).double().numpy()
        ref, _ = sample(xc[b].numpy(), np.arange(32)[None, :] + dx * 16, np.arange(28)[:, None] + dy * 14, False, 0.25)
        assert np.array_equal(out[b].double().numpy(), ref), b


# ---- the draws --------------------------------------------------------------------------------------------------------------

def test_noise_is_uniform_and_independent():
    from scipy import stats

    x = torch.zeros(256, 1, 28, 28, device=dev())
    torch.manual_seed(1234)
    t = pdt.data.ElasticTransform(record_params=True)
    calls = []
    for _ in range(3):
        t(x)
        calls.append(t.last_params.cpu().double().numpy())
    v = np.concatenate([c.ravel() for c in calls])
    assert v.min() >= -1.0 and v.max() < 1.0
    assert stats.kstest(v, stats.uniform(loc=-1.0, scale=2.0).cdf).pvalue > 1e-3
    # correlation between planes of different images, between the two planes of one image, and between consecutive calls
    n = 28 * 28
    bound = 5 / math.sqrt(n)
    c0, c1 = calls[0], calls[1]
    pairs = [(c0[i, 0], c0[i + 1, 0]) for i in range(0, 255, 8)] + [(c0[i, 0], c0[i, 1]) for i in range(0, 256, 8)]
    pairs += [(c0[i, 0], c1[i, 0]) for i in range(0, 256, 8)]
    for a, b in pairs:
        assert abs(np.corrcoef(a.ravel(), b.ravel())[0, 1]) < bound
    torch.manual_seed(1234)
    t(x)
    assert np.array_equal(t.last_params.cpu().double().numpy(), calls[0])   # manual_seed reproduces the draws


@pytest.mark.parametrize("own_generator", [False, True])
def test_graph_replays_draw_and_reseed(own_generator):
    x = torch.rand(64, 1, 28, 28, generator=torch.Generator().manual_seed(6)).to(dev())
    gen = torch.Generator(device=dev()) if own_generator else None
    seed = (lambda s: gen.manual_seed(s)) if own_generator else torch.manual_seed
    t = pdt.data.ElasticTransform(34.0, 4.0, record_params=True, generator=gen)
    seed(5)
    e1, p1 = t(x).clone(), t.last_params.clone()
    e2, p2 = t(x).clone(), t.last_params.clone()
    seed(5)
    assert torch.equal(t(x), e1) and torch.equal(t.last_params, p1)
    g = torch.cuda.CUDAGraph()
    if own_generator:
        g.register_generator_state(gen)
    with torch.cuda.graph(g):
        out = t(x)
    noise = t.last_params
    seed(5)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, e1) and torch.equal(noise, p1)   # a replay draws what the eager call drew from the same seed
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, e2) and torch.equal(noise, p2)   # consecutive replays draw new values, as consecutive calls do
    assert (p1 == p2).float().mean().item() < 1e-3
    seed(5)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, e1)


def test_capture_before_first_call_is_refused():
    t = pdt.data.ElasticTransform()
    x = torch.rand(4, 1, 28, 28, device=dev())
    g = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="before capturing"):
        with torch.cuda.graph(g):
            t(x)


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


def test_zero_alpha_step_changes_nothing():
    with _one_gpu():
        xs = _batches(3, 100)
        plain_model, plain = _step(None)
        aug_model, aug = _step(pdt.data.ElasticTransform(alpha=0.0))
        assert plain.kernels_per_replay == 3 and aug.kernels_per_replay == 4, (plain.kernels_per_replay, aug.kernels_per_replay)
        for r in range(6):
            la, lb = plain(*xs[r % 3]), aug(*xs[r % 3])
            torch.cuda.synchronize()
            assert torch.equal(la, lb), (r, la.item(), lb.item())
        for (n, p), q in zip(plain_model.named_parameters(), aug_model.parameters()):
            assert torch.equal(p, q), n
        for b, c in zip(plain_model.buffers(), aug_model.buffers()):
            assert torch.equal(b, c)


def test_affine_then_elastic_step_matches_forward_of_rebuilt_batch():
    """[RandomAffine, ElasticTransform] in one graphed step: 5 launches, both transforms' last_params are the replayed graph's records,
    and the loss equals the forward of the batch rebuilt in float64 from them."""
    with _one_gpu():
        xs = _batches(3, 100)
        gen = torch.Generator(device=dev())
        affine = pdt.data.RandomAffine(0, translate=(0.15, 0.15), record_params=True, generator=gen)
        elastic = pdt.data.ElasticTransform(34.0, 4.0, record_params=True, generator=gen)
        model, step = _step([affine, elastic])
        assert step.kernels_per_replay == 5, step.kernels_per_replay
        gen.manual_seed(3)
        seen = []
        for r in range(6):
            ref = pdt.models.ConvNet().to(dev())
            ref.load_state_dict(model.state_dict())   # the model before this step's update
            x, y = xs[r % 3]
            loss = step(x, y)
            torch.cuda.synchronize()
            p, n = affine.last_params.cpu(), elastic.last_params.cpu()
            seen.append((p.clone(), n.clone()))
            xc = x.cpu().numpy()
            rebuilt = np.empty_like(xc, dtype=np.float64)
            for b in range(x.shape[0]):
                shifted, _ = affine_reference(xc[b], p[b].numpy(), False, 0.0)   # integer shifts: exact
                sx, sy, _ = source_coords(n[b].numpy(), elastic.alpha, elastic.sigma)
                rebuilt[b], _ = sample(shifted, sx, sy, True, 0.0)
            with torch.no_grad():
                expect = F.cross_entropy(ref(torch.from_numpy(rebuilt).float().to(dev())).double(), y)
            assert abs(loss.item() - expect.item()) <= 1e-4 * abs(expect.item()), (r, loss.item(), expect.item())
        for (pa, na), (pb, nb) in zip(seen, seen[1:]):
            assert not torch.equal(pa, pb) and not torch.equal(na, nb)   # every replay draws new parameters and fields
        # one generator: the affine's launch advances the offset before the elastic one draws, so neither repeats the other's values
        gen.manual_seed(3)
        step(*xs[0])
        torch.cuda.synchronize()
        assert torch.equal(affine.last_params.cpu(), seen[0][0]) and torch.equal(elastic.last_params.cpu(), seen[0][1])


def test_accumulation_augments_all_rows_once():
    with _one_gpu():
        t = pdt.data.ElasticTransform(record_params=True)
        model, step = _step(t, k=2)
        assert step.kernels_per_replay == 3 * 2 + 1, step.kernels_per_replay
        xs = _batches(2, 200)
        for r in range(4):
            loss = step(*xs[r % 2])
            torch.cuda.synchronize()
            assert math.isfinite(loss.item())
            n = t.last_params
            assert n.shape == (200, 2, 28, 28)
            assert len(set(n[:, 0, 0, 0].tolist())) > 195   # every row drew its own field


def test_train_script_with_affine_and_elastic_in_graphed_step():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "1", "--graph", "--rotate", "10", "--translate", "0.1",
                          "--elastic-alpha", "34", "--elastic-sigma", "4", "--cutmix", "1.0", "--steps", "20", "--samples", "4000",
                          "--epochs", "1", "--log-interval", "5", "--eval"],
                         capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    losses = [float(v) for v in re.findall(r"Step \[\d+/\d+\], Loss: (\S+)", out.stdout)]
    assert len(losses) == 4 and all(math.isfinite(v) for v in losses), out.stdout[-1000:]
    assert re.search(r"Test Loss: \S+, Accuracy: \S+% \(10000 images\)", out.stdout), out.stdout[-1000:]
