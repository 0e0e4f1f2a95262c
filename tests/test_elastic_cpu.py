"""pdt.data.ElasticTransform without a GPU: torchvision's argument rules and call-time errors, the CPU path against a float64
reference of torchvision's definition rebuilt from the recorded noise (and torchvision itself when it is importable), the exact
cases, the draws against a per-image torchvision loop, and train_mnist.py's elastic flags.

The reference (also used by test_elastic.py on the GPU) blurs the recorded noise in float64 with torchvision's fp32 1-D weights
(reflect padding, x then y), scales it by alpha / (W, H) and samples the image at (j + dx·W/2, i + dy·H/2) with the float64 taps of
test_random_affine_cpu.py.  Tolerances:
  * bilinear: the first-order rounding bound of an fp32 blur that sums its taps in order (u·Σ|partial sums| per pass, u = 2^-24),
    plus the fp32 scaling, times alpha/2 pixels per unit, times the image's largest step between samples, plus 16u for the
    sampling's own rounding.  About 1e-5 for images in [0, 1] at alpha 50, sigma 5.
  * nearest: bit-equal except where the float64 source coordinate lies within 1e-4 of a rounding tie (x.5); the test asserts that
    the source-coordinate bound stays below that band."""
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import pytorch_distributed_train_b200 as pdt
from pytorch_distributed_train_b200 import cli
from test_random_affine_cpu import HALF_BAND

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24

try:
    from torchvision.transforms import v2 as TV
    from torchvision.transforms.v2 import functional as TVF
except Exception:   # noqa: BLE001  (torchvision is optional)
    TV = TVF = None


def kernel_size(sigma):
    k = int(8 * sigma + 1)
    return k + 1 if k % 2 == 0 else k


def gaussian1d(k, sigma):
    """torchvision's _get_gaussian_kernel1d in fp32, as float64 numbers."""
    lim = (k - 1) / (2.0 * math.sqrt(2.0))
    x = torch.linspace(-lim, lim, steps=k, dtype=torch.float32)
    return torch.softmax(x.div(sigma).pow(2).neg(), dim=0).double().numpy()


def blur(v, k, sigma):
    """float64 separable blur of v [H, W] (reflect padding k // 2; x weights (k, sigma[0]), y weights (k, sigma[1])) and the
    first-order bound of the rounding error of the same blur in fp32 with its taps summed in order."""
    wx, wy = gaussian1d(k, sigma[0]), gaussian1d(k, sigma[1])
    r = k // 2
    H, W = v.shape
    pv = np.pad(v, ((0, 0), (r, r)), mode="reflect")
    part = np.cumsum(np.stack([wx[t] * pv[:, t:t + W] for t in range(k)], -1), -1)
    h, eh = part[..., -1], U * np.abs(part).sum(-1)
    ph, peh = np.pad(h, ((r, r), (0, 0)), mode="reflect"), np.pad(eh, ((r, r), (0, 0)), mode="reflect")
    part = np.cumsum(np.stack([wy[t] * ph[t:t + H] for t in range(k)], -1), -1)
    err = sum(wy[t] * peh[t:t + H] for t in range(k)) + U * np.abs(part).sum(-1)
    return part[..., -1], err


def source_coords(noise, alpha, sigma):
    """float64 source coordinates (sx, sy) [H, W] from one image's recorded noise [2, H, W], and the bound of their fp32 error."""
    noise = np.asarray(noise, dtype=np.float64)
    _, H, W = noise.shape
    disp, errs = [], []
    for c, size in ((0, W), (1, H)):
        v, e = noise[c], np.zeros((H, W))
        if sigma[c] > 0:
            v, e = blur(v, kernel_size(sigma[c]), sigma)
        disp.append(v * alpha[c] / size)
        errs.append(abs(alpha[c]) / 2 * (e + 2 * U * np.abs(v)))   # in pixels: (W/2)·(alpha/W)·(blur error + the two roundings)
    sx = np.arange(W, dtype=np.float64)[None, :] + disp[0] * (W / 2)
    sy = np.arange(H, dtype=np.float64)[:, None] + disp[1] * (H / 2)
    return sx, sy, errs[0] + errs[1]


def sample(img, sx, sy, bilinear, fill):
    """float64 [C, H, W] of img sampled at (sx, sy), and the [H, W] mask of pixels whose nearest tap is ambiguous."""
    img = np.asarray(img, dtype=np.float64)
    C, H, W = img.shape

    def tap(ix, iy):
        inside = (ix >= 0) & (ix <= W - 1) & (iy >= 0) & (iy <= H - 1)
        v = img[:, np.where(inside, iy, 0).astype(np.int64), np.where(inside, ix, 0).astype(np.int64)]
        return inside, np.where(inside[None], v, 0.0)

    ambiguous = (np.abs(sx - np.floor(sx) - 0.5) < HALF_BAND) | (np.abs(sy - np.floor(sy) - 0.5) < HALF_BAND)
    if not bilinear:
        inside, v = tap(np.rint(sx), np.rint(sy))
        return np.where(inside[None], v, fill), ambiguous
    x0, y0 = np.floor(sx), np.floor(sy)
    fx, fy = sx - x0, sy - y0
    acc, mask = np.zeros((C, H, W)), np.zeros((H, W))
    for dx, dy, w in ((0, 0, (1 - fx) * (1 - fy)), (1, 0, fx * (1 - fy)), (0, 1, (1 - fx) * fy), (1, 1, fx * fy)):
        inside, v = tap(x0 + dx, y0 + dy)
        w = np.where(inside, w, 0.0)
        acc += w[None] * v
        mask += w
    return (acc - fill) * mask[None] + fill, ambiguous


def check_against_reference(x, out, noise, alpha, sigma, bilinear, fill):
    """Every image of out against the float64 reference rebuilt from its recorded noise; returns the largest bilinear tolerance
    used (0 for nearest)."""
    x, out, noise = x.cpu().double().numpy(), out.cpu().double().numpy(), noise.cpu().double().numpy()
    worst_tol = 0.0
    for b in range(x.shape[0]):
        sx, sy, err = source_coords(noise[b], alpha, sigma)
        assert err.max() < HALF_BAND, err.max()
        ref, ambiguous = sample(x[b], sx, sy, bilinear, fill)
        if bilinear:
            span = max(x[b].max(), fill) - min(x[b].min(), fill)   # the largest step of the interpolant per unit of either coordinate
            tol = span * err.max() + 16 * U * max(np.abs(x[b]).max(), abs(fill), 1.0)
            worst_tol = max(worst_tol, tol)
            assert np.abs(out[b] - ref).max() <= tol, (b, np.abs(out[b] - ref).max(), tol)
        else:
            diff = (out[b] != ref).any(0)
            assert not (diff & ~ambiguous).any(), (b, np.argwhere(diff & ~ambiguous)[:5])
    return worst_tol


def torchvision_displacement(noise, alpha, sigma):
    """torchvision's make_params from the recorded noise [2, H, W] (fp32): its gaussian_blur and scaling, [1, H, W, 2]."""
    _, H, W = noise.shape
    planes = []
    for c, size in ((0, W), (1, H)):
        d = noise[c].view(1, 1, H, W)
        if sigma[c] > 0:
            k = kernel_size(sigma[c])
            d = TVF.gaussian_blur(d, [k, k], list(sigma))
        planes.append(d * alpha[c] / size)
    return torch.cat(planes, 1).permute([0, 2, 3, 1])


def check_against_torchvision(x, out, noise, alpha, sigma, bilinear, fill, tol):
    """Every image of out against torchvision's F.elastic fed the displacement of the recorded noise; torchvision forms its grid in
    fp32, which adds up to a few W·u to the source coordinate."""
    xc, oc, nc = x.cpu(), out.cpu(), noise.cpu()
    mode = TVF.InterpolationMode.BILINEAR if bilinear else TVF.InterpolationMode.NEAREST
    for b in range(xc.shape[0]):
        tv = TVF.elastic(xc[b], torchvision_displacement(nc[b], alpha, sigma), interpolation=mode, fill=fill)
        if bilinear:
            W = xc.shape[-1]
            assert (oc[b] - tv).abs().max().item() <= tol + 8 * W * U, b
        else:
            sx, sy, _ = source_coords(nc[b].numpy(), alpha, sigma)
            _, ambiguous = sample(xc[b].numpy(), sx, sy, False, fill)
            diff = (oc[b] != tv).any(0).numpy()
            assert not (diff & ~ambiguous).any(), b


# ---- arguments ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kwargs, err, msg", [
    (dict(alpha=None), TypeError, "alpha should be a number or a sequence of numbers. Got <class 'NoneType'>"),
    (dict(alpha=(1.0, 2.0, 3.0)), ValueError, "If alpha is a sequence its length should be 1 or 2. Got 3"),
    (dict(alpha=(1.0, "a")), ValueError, "alpha should be a sequence of numbers. Got <class 'str'>"),
    (dict(sigma={1: 2}), TypeError, "sigma should be a number or a sequence of numbers. Got <class 'dict'>"),
    (dict(sigma=()), ValueError, "If sigma is a sequence its length should be 1 or 2. Got 0"),
    (dict(sigma=[None]), ValueError, "sigma should be a sequence of numbers. Got <class 'NoneType'>"),
    (dict(interpolation="bicubic"), ValueError, "Interpolation mode 'bicubic' is unsupported with Tensor input"),
])
def test_arguments_follow_torchvision(kwargs, err, msg):
    with pytest.raises(err, match="^" + re.escape(msg) + "$"):
        pdt.data.ElasticTransform(**kwargs)
    if TV is not None and "interpolation" not in kwargs:   # torchvision refuses strings for interpolation altogether
        with pytest.raises(err, match="^" + re.escape(msg) + "$"):
            TV.ElasticTransform(**kwargs)


@pytest.mark.parametrize("sigma, shape, err, msg", [
    ((5.0, 0.0), (2, 1, 28, 28), ValueError, "sigma should have positive values. Got [5.0, 0.0]"),
    ((-1.0, 3.0), (2, 1, 28, 28), ValueError, "sigma should have positive values. Got [-1.0, 3.0]"),
    (7.0, (2, 1, 28, 28), RuntimeError, "Argument #4: Padding size should be less than the corresponding input dimension, but got: "
                                        "padding (28, 28) at dimension 3 of input [1, 1, 28, 28]"),
    (3.0, (2, 1, 10, 36), RuntimeError, "Argument #6: Padding size should be less than the corresponding input dimension, but got: "
                                        "padding (12, 12) at dimension 2 of input [1, 1, 10, 36]"),
    ((1.0, 5.0), (1, 2, 28, 16), RuntimeError, "Argument #4: Padding size should be less than the corresponding input dimension, but "
                                               "got: padding (20, 20) at dimension 3 of input [1, 1, 28, 16]"),
])
def test_call_time_errors_follow_torchvision(sigma, shape, err, msg):
    t = pdt.data.ElasticTransform(sigma=sigma)   # accepted until it meets an image, as torchvision's
    with pytest.raises(err, match="^" + re.escape(msg) + "$"):
        t(torch.rand(shape))
    if TV is not None:
        tv = TV.ElasticTransform(sigma=sigma)
        with pytest.raises(err, match="^" + re.escape(msg) + "$"):
            tv(torch.rand(shape[1:]))


def test_arguments_normalised_like_torchvision():
    t = pdt.data.ElasticTransform()
    assert t.alpha == [50.0, 50.0] and t.sigma == [5.0, 5.0] and t.interpolation == "bilinear" and t.fill == 0.0
    t = pdt.data.ElasticTransform((3,), [1, 2], interpolation="nearest", fill=1)
    assert t.alpha == [3.0, 3.0] and t.sigma == [1.0, 2.0] and t.interpolation == "nearest" and t.fill == 1.0
    if TVF is not None:
        assert pdt.data.ElasticTransform(interpolation=TVF.InterpolationMode.NEAREST).interpolation == "nearest"
        tv = TV.ElasticTransform((3,), [1, 2])
        assert tv.alpha == t.alpha and tv.sigma == t.sigma
    with pytest.raises(TypeError):
        pdt.data.ElasticTransform(fill=(1, 2, 3))


def test_weights_equal_torchvision_bit_for_bit():
    for sigma in ((5.0, 5.0), (4.0, 1.0), (0.3, 2.5)):
        t = pdt.data.ElasticTransform(sigma=sigma)
        kx, ky = kernel_size(sigma[0]), kernel_size(sigma[1])
        parts = [gaussian1d(kx, sigma[0]), gaussian1d(kx, sigma[1]), gaussian1d(ky, sigma[0]), gaussian1d(ky, sigma[1])]
        assert torch.equal(t._host_weights.double(), torch.from_numpy(np.concatenate(parts)))
        if TVF is not None:
            from torchvision.transforms.v2.functional._misc import _get_gaussian_kernel1d

            for k, s in ((kx, sigma[0]), (ky, sigma[1])):
                assert torch.equal(torch.from_numpy(gaussian1d(k, s)).float(), _get_gaussian_kernel1d(k, s, torch.float32, torch.device("cpu")))


def test_other_dtypes_and_shapes_refused():
    t = pdt.data.ElasticTransform()
    for dt in (torch.float64, torch.float16, torch.uint8):
        with pytest.raises(TypeError):
            t(torch.zeros(2, 1, 28, 28, dtype=dt))
    with pytest.raises(ValueError):
        t(torch.zeros(1, 28, 28))


# ---- the CPU path against float64 -----------------------------------------------------------------------------------------------

CASES = [   # (shape, alpha, sigma)
    ((16, 1, 28, 28), 50.0, 5.0),
    ((6, 3, 32, 32), 34.0, 4.0),
    ((6, 1, 20, 36), 20.0, (4.0, 1.0)),
    ((6, 3, 28, 28), (30.0, 10.0), (1.0, 4.0)),
    ((6, 1, 28, 28), 8.0, 1.0),
    ((6, 2, 24, 30), 40.0, 0.0),
    ((0, 1, 28, 28), 50.0, 5.0),
]


@pytest.mark.parametrize("shape, alpha, sigma", CASES)
@pytest.mark.parametrize("interpolation", ["nearest", "bilinear"])
@pytest.mark.parametrize("fill", [0.0, 0.5])
def test_cpu_path_matches_float64_reference(shape, alpha, sigma, interpolation, fill):
    x = torch.rand(shape, generator=torch.Generator().manual_seed(3))
    t = pdt.data.ElasticTransform(alpha, sigma, interpolation=interpolation, fill=fill, generator=torch.Generator().manual_seed(11),
                                  record_params=True)
    out = t(x)
    assert out.shape == x.shape and out.dtype == torch.float32 and t.last_params.shape == (shape[0], 2) + shape[2:]
    tol = check_against_reference(x, out, t.last_params, t.alpha, t.sigma, interpolation == "bilinear", fill)
    assert tol <= 5e-5, tol
    if TVF is not None and shape[0]:
        check_against_torchvision(x, out, t.last_params, t.alpha, t.sigma, interpolation == "bilinear", fill, tol)


def test_cpu_exact_cases():
    x = torch.rand(5, 2, 28, 28)
    for interpolation in ("nearest", "bilinear"):
        for sigma in (5.0, 0.0):
            assert torch.equal(pdt.data.ElasticTransform(0.0, sigma, interpolation=interpolation)(x), x)
    empty = torch.rand(0, 1, 28, 28)
    out = pdt.data.ElasticTransform()(empty)
    assert out.shape == empty.shape and out is not empty


def test_cpu_unblurred_displacement_is_exact():
    """sigma <= 0: no blur, the displacement is fl(fl(noise·alpha)/W) and the nearest output is bit-equal everywhere."""
    x = torch.rand(8, 1, 28, 32)
    t = pdt.data.ElasticTransform(37.3, 0.0, interpolation="nearest", fill=0.25, record_params=True)
    out = t(x)
    n = t.last_params
    for b in range(8):
        dx, dy = (n[b, 0] * 37.3 / 32).double().numpy(), (n[b, 1] * 37.3 / 28).double().numpy()
        sx, sy = np.arange(32)[None, :] + dx * 16, np.arange(28)[:, None] + dy * 14
        ref, _ = sample(x[b].numpy(), sx, sy, False, 0.25)
        assert np.array_equal(out[b].double().numpy(), ref), b


def test_cpu_draws_match_a_torchvision_loop():
    x = torch.rand(5, 1, 28, 28)
    torch.manual_seed(21)
    t = pdt.data.ElasticTransform(record_params=True)
    t(x)
    torch.manual_seed(21)
    expect = torch.stack([torch.cat([torch.rand(1, 1, 28, 28) * 2 - 1 for _ in range(2)], 1)[0] for _ in range(5)])
    assert torch.equal(t.last_params, expect)
    if TV is not None:
        torch.manual_seed(21)
        tv = TV.ElasticTransform()
        for b in range(5):
            disp = tv.make_params([x[b]])["displacement"]
            assert torch.equal(disp, torchvision_displacement(t.last_params[b], tv.alpha, tv.sigma)), b


def test_cpu_generator_reproduces():
    x = torch.rand(4, 1, 28, 28)
    a = pdt.data.ElasticTransform(generator=torch.Generator().manual_seed(5))(x)
    assert torch.equal(pdt.data.ElasticTransform(generator=torch.Generator().manual_seed(5))(x), a)
    torch.manual_seed(9)
    c = pdt.data.ElasticTransform()(x)
    torch.manual_seed(9)
    assert torch.equal(pdt.data.ElasticTransform()(x), c)
    assert not torch.equal(c, a)


# ---- the CLI --------------------------------------------------------------------------------------------------------------------

def test_cli_parses_elastic_flags():
    p = cli.build_parser()
    a = p.parse_args([])
    assert a.elastic_alpha is None and a.elastic_sigma is None and cli.make_elastic(a, None) is None
    a = p.parse_args(["--elastic-alpha", "34"])
    cli.check_args(p, a)
    t = cli.make_elastic(a, torch.Generator())
    assert t.alpha == [34.0, 34.0] and t.sigma == [5.0, 5.0] and t.interpolation == "bilinear"
    a = p.parse_args(["--elastic-alpha", "20", "--elastic-sigma", "4", "--rotate", "10", "--cutmix", "1.0"])
    cli.check_args(p, a)
    gen = torch.Generator()
    t = cli.make_elastic(a, gen)
    assert t.sigma == [4.0, 4.0] and t.generator is gen and cli.make_augment(a, gen).generator is gen


@pytest.mark.parametrize("flags, msg", [
    (["--elastic-sigma", "4"], "--elastic-sigma needs --elastic-alpha"),
    (["--elastic-alpha", "30", "--mixup", "0.2"], "--mixup cannot be combined with --elastic-alpha"),
])
def test_cli_refuses_bad_elastic_flags(flags, msg):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py")] + flags, capture_output=True, text=True, timeout=60,
                         cwd=ROOT)
    assert out.returncode != 0 and msg in out.stderr, out.stderr[-500:]


@pytest.mark.parametrize("ranks, extra", [(1, []), (2, ["--rotate", "10", "--translate", "0.1"]), (1, ["--rotate", "10", "--cutmix", "1.0",
                                                                                                         "--accumulation-steps", "2",
                                                                                                         "--ema-decay", "0.9", "--eval"])])
def test_train_script_runs_with_elastic_on_gloo(ranks, extra):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", str(ranks), "--backend", "gloo", "--epochs", "1",
                          "--steps", "3", "--elastic-alpha", "34", "--log-interval", "1", "--samples", "2000", "--batch-size", "50"] + extra,
                         capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-1500:] + out.stderr[-1500:]
    losses = [float(v) for v in re.findall(r"Step \[\d+/\d+\], Loss: (\S+)", out.stdout)]
    assert len(losses) == 3 and all(math.isfinite(v) for v in losses), out.stdout[-1500:]
    if "--eval" in extra:
        assert re.search(r"Test Loss: \S+, Accuracy: \S+% \(10000 images\)", out.stdout), out.stdout[-1000:]


def test_resumed_run_draws_the_uninterrupted_elastic_sequence(tmp_path):
    """The affine and elastic transforms share a generator seeded from (epoch, rank), so a run resumed from an epoch's checkpoint
    trains epoch 2 on the images an uninterrupted run warps."""
    base = [sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "1", "--backend", "gloo", "--rotate", "15", "--elastic-alpha", "34",
            "--elastic-sigma", "4", "--steps", "3", "--samples", "400", "--log-interval", "1"]

    def run(*extra):
        out = subprocess.run(base + list(extra), capture_output=True, text=True, timeout=240, cwd=ROOT)
        assert out.returncode == 0, out.stderr[-2000:]
        return re.findall(r"Epoch \[2/2\], Step \[\d+/\d+\], Loss: \S+", out.stdout)

    ck = str(tmp_path / "run.pt")
    whole = run("--epochs", "2")
    run("--epochs", "1", "--checkpoint", ck)
    resumed = run("--epochs", "2", "--resume", ck)
    assert len(whole) == 3 and resumed == whole, (whole, resumed)
