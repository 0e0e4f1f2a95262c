"""pdt.data.RandomAffine without a GPU: torchvision's argument rules, the CPU path against a float64 reference of torchvision's
definition (and torchvision itself when it is importable), the exact cases, and train_mnist.py's augmentation flags.

The reference (also used by test_random_affine.py on the GPU) is torchvision's _get_inverse_affine_matrix with center (0, 0),
the source coordinate of output pixel (i, j)
    sx = m0·(j − cw) + m1·(i − ch) + m2 + cw,   sy = m3·(j − cw) + m4·(i − ch) + m5 + ch,   cw = (W − 1)/2, ch = (H − 1)/2
and numpy taps, all in float64.  Tolerances: bilinear within 1e-5 on inputs in [0, 1]; nearest bit-equal except where a source
coordinate lies within 1e-4 of a rounding boundary (x.5), where fp32 and float64 may round to different pixels.  torchvision's own
fp32 output sits within 4.5e-6 (bilinear) of this reference, with no nearest mismatch outside that band."""
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BILINEAR_TOL = 1e-5
HALF_BAND = 1e-4

try:
    from torchvision.transforms.v2 import functional as TVF
except Exception:   # noqa: BLE001  (torchvision is optional)
    TVF = None


def inverse_matrix(angle, tx, ty, scale, shear_x, shear_y):
    """torchvision's _get_inverse_affine_matrix(center=[0, 0], angle, (tx, ty), scale, (shear_x, shear_y)), in float64."""
    rot, sx, sy = math.radians(angle), math.radians(shear_x), math.radians(shear_y)
    a = math.cos(rot - sy) / math.cos(sy)
    b = -math.cos(rot - sy) * math.tan(sx) / math.cos(sy) - math.sin(rot)
    c = math.sin(rot - sy) / math.cos(sy)
    d = -math.sin(rot - sy) * math.tan(sx) / math.cos(sy) + math.cos(rot)
    m = [x / scale for x in [d, -b, 0.0, -c, a, 0.0]]
    m[2] += m[0] * -tx + m[1] * -ty
    m[5] += m[3] * -tx + m[4] * -ty
    return m


def source_coords(params, H, W):
    """float64 source coordinates (sx, sy) [H, W] of one image's parameters (angle, tx, ty, scale, shear_x, shear_y)."""
    m = inverse_matrix(*[float(v) for v in params])
    cw, ch = (W - 1) / 2, (H - 1) / 2
    j = np.arange(W, dtype=np.float64)[None, :] - cw
    i = np.arange(H, dtype=np.float64)[:, None] - ch
    return m[0] * j + m[1] * i + m[2] + cw, m[3] * j + m[4] * i + m[5] + ch


def reference(img, params, bilinear, fill):
    """float64 [C, H, W] of one image, and the [H, W] mask of pixels whose nearest tap is ambiguous (within HALF_BAND of x.5)."""
    img = np.asarray(img, dtype=np.float64)
    C, H, W = img.shape
    sx, sy = source_coords(params, H, W)

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


def check_against_reference(x, out, params, bilinear, fill):
    """Every image of out against the float64 reference of its recorded parameters; returns how many nearest pixels fell in the
    ambiguous band and differed."""
    x, out, params = x.cpu().double().numpy(), out.cpu().double().numpy(), params.cpu().double().numpy()
    banded = 0
    for b in range(x.shape[0]):
        ref, ambiguous = reference(x[b], params[b], bilinear, fill)
        if bilinear:
            err = np.abs(out[b] - ref).max()
            assert err <= BILINEAR_TOL, (b, err, params[b])
        else:
            diff = (out[b] != ref).any(0)
            assert not (diff & ~ambiguous).any(), (b, params[b], np.argwhere(diff & ~ambiguous)[:5])
            banded += int(diff.sum())
    return banded


def torchvision_affine(img, params, bilinear, fill):
    angle, tx, ty, scale, shx, shy = [float(v) for v in params]
    return TVF.affine(img, angle=angle, translate=[int(tx), int(ty)], scale=scale, shear=[shx, shy],
                      interpolation=TVF.InterpolationMode.BILINEAR if bilinear else TVF.InterpolationMode.NEAREST, fill=fill)


def check_against_torchvision(x, out, params, bilinear, fill):
    """Every image of out against torchvision.transforms.v2.functional.affine with its recorded parameters, at the same tolerances."""
    xc, oc, pc = x.cpu(), out.cpu(), params.cpu()
    for b in range(xc.shape[0]):
        tv = torchvision_affine(xc[b], pc[b], bilinear, fill)
        if bilinear:
            assert (oc[b] - tv).abs().max().item() <= BILINEAR_TOL, (b, pc[b])
        else:
            _, ambiguous = reference(xc[b].numpy(), pc[b].numpy(), False, fill)
            diff = (oc[b] != tv).any(0).numpy()
            assert not (diff & ~ambiguous).any(), (b, pc[b])


# ---- arguments ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kwargs, err, msg", [
    (dict(degrees=-1), ValueError, "If degrees is a single number, it must be positive."),
    (dict(degrees=(1, 2, 3)), ValueError, "degrees should be a sequence of length 2."),
    (dict(degrees=10, translate=0.1), TypeError, "translate should be a sequence of length 2."),
    (dict(degrees=10, translate=(0.1,)), ValueError, "translate should be a sequence of length 2."),
    (dict(degrees=10, translate=(0.1, 1.5)), ValueError, "translation values should be between 0 and 1"),
    (dict(degrees=10, scale=(0.0, 1.0)), ValueError, "scale values should be positive"),
    (dict(degrees=10, scale=1.0), TypeError, "scale should be a sequence of length 2."),
    (dict(degrees=10, shear=-5), ValueError, "If shear is a single number, it must be positive."),
    (dict(degrees=10, shear=(1, 2, 3)), ValueError, "shear should be a sequence of length 2 or 4."),
    (dict(degrees=10, interpolation="bicubic"), ValueError, "Interpolation mode 'bicubic' is unsupported with Tensor input"),
])
def test_arguments_follow_torchvision(kwargs, err, msg):
    with pytest.raises(err, match="^" + re.escape(msg) + "$"):
        pdt.data.RandomAffine(**kwargs)
    if TVF is not None:
        from torchvision.transforms import v2

        tv_kwargs = dict(kwargs)
        if "interpolation" in tv_kwargs:
            return   # torchvision refuses strings for interpolation altogether
        with pytest.raises(err, match="^" + re.escape(msg) + "$"):
            v2.RandomAffine(**tv_kwargs)


def test_arguments_normalised_like_torchvision():
    t = pdt.data.RandomAffine(15, (0.1, 0.2), (0.9, 1.1), 5)
    assert t.degrees == [-15.0, 15.0] and t.translate == [0.1, 0.2] and t.scale == [0.9, 1.1] and t.shear == [-5.0, 5.0]
    assert pdt.data.RandomAffine((2, 3), shear=(1, 2, 3, 4)).shear == [1.0, 2.0, 3.0, 4.0]
    assert pdt.data.RandomAffine(0).interpolation == "nearest"
    if TVF is not None:
        assert pdt.data.RandomAffine(0, interpolation=TVF.InterpolationMode.BILINEAR).interpolation == "bilinear"


def test_other_dtypes_refused():
    t = pdt.data.RandomAffine(10)
    for dt in (torch.float64, torch.float16, torch.uint8):
        with pytest.raises(TypeError):
            t(torch.zeros(2, 1, 4, 4, dtype=dt))
    with pytest.raises(ValueError):
        t(torch.zeros(1, 4, 4))


# ---- the CPU path against float64 -----------------------------------------------------------------------------------------------

SHAPES = [(100, 1, 28, 28), (7, 3, 32, 48), (0, 1, 28, 28)]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("interpolation", ["nearest", "bilinear"])
@pytest.mark.parametrize("fill", [0.0, 0.5])
def test_cpu_path_matches_float64_reference(shape, interpolation, fill):
    g = torch.Generator().manual_seed(3)
    x = torch.rand(shape, generator=g)
    t = pdt.data.RandomAffine(25, (0.15, 0.1), (0.8, 1.2), (-10, 10, -5, 5), interpolation=interpolation, fill=fill,
                              generator=torch.Generator().manual_seed(11), record_params=True)
    out = t(x)
    assert out.shape == x.shape and out.dtype == torch.float32 and t.last_params.shape == (shape[0], 6)
    check_against_reference(x, out, t.last_params, interpolation == "bilinear", fill)
    if TVF is not None and shape[0]:
        check_against_torchvision(x, out, t.last_params, interpolation == "bilinear", fill)


def test_cpu_path_draws_follow_the_ranges():
    t = pdt.data.RandomAffine((-20, 30), (0.1, 0.2), (0.5, 2.0), (1, 2, 3, 4), generator=torch.Generator().manual_seed(0),
                              record_params=True)
    t(torch.zeros(4096, 1, 28, 20))
    p = t.last_params
    assert p[:, 0].min() >= -20 and p[:, 0].max() < 30
    assert (p[:, 1] == p[:, 1].round()).all() and p[:, 1].abs().max() <= round(0.1 * 20)
    assert (p[:, 2] == p[:, 2].round()).all() and p[:, 2].abs().max() <= round(0.2 * 28)
    assert p[:, 3].min() >= 0.5 and p[:, 3].max() < 2.0
    assert p[:, 4].min() >= 1 and p[:, 4].max() < 2 and p[:, 5].min() >= 3 and p[:, 5].max() < 4
    assert len(set(p[:, 0].tolist())) > 4000


def test_cpu_exact_cases():
    x = torch.rand(5, 2, 28, 28)
    # torchvision's positive angles turn the picture counter-clockwise on screen: x toward -y, which is rot90 from W towards H
    assert torch.equal(pdt.data.RandomAffine((90, 90))(x), torch.rot90(x, 1, (-1, -2)))
    assert torch.equal(pdt.data.RandomAffine(0)(x), x)
    assert torch.equal(pdt.data.RandomAffine(0, interpolation="bilinear")(x), x)
    t = pdt.data.RandomAffine(0, translate=(0.2, 0.2), fill=0.25, record_params=True)
    out = t(x)
    for b in range(5):
        tx, ty = int(t.last_params[b, 1]), int(t.last_params[b, 2])
        ref = torch.full_like(x[b], 0.25)
        ref[:, max(ty, 0):28 + min(ty, 0), max(tx, 0):28 + min(tx, 0)] = x[b][:, max(-ty, 0):28 + min(-ty, 0), max(-tx, 0):28 + min(-tx, 0)]
        assert torch.equal(out[b], ref), (tx, ty)


def test_cpu_generator_reproduces():
    x = torch.rand(8, 1, 28, 28)
    a = pdt.data.RandomAffine(30, (0.1, 0.1), generator=torch.Generator().manual_seed(5))(x)
    b = pdt.data.RandomAffine(30, (0.1, 0.1), generator=torch.Generator().manual_seed(5))(x)
    assert torch.equal(a, b)
    torch.manual_seed(9)
    c = pdt.data.RandomAffine(30)(x)
    torch.manual_seed(9)
    assert torch.equal(pdt.data.RandomAffine(30)(x), c)


# ---- the CLI --------------------------------------------------------------------------------------------------------------------

def test_cli_parses_augmentation_flags():
    p = cli.build_parser()
    a = p.parse_args([])
    assert a.rotate is None and a.translate is None and a.scale_range is None and a.shear is None and a.affine_interpolation == "nearest"
    assert cli.make_augment(a, None) is None
    a = p.parse_args(["--rotate", "10", "--translate", "0.1", "--scale-range", "0.9", "1.1", "--shear", "5",
                      "--affine-interpolation", "bilinear"])
    cli.check_args(p, a)
    t = cli.make_augment(a, torch.Generator())
    assert t.degrees == [-10.0, 10.0] and t.translate == [0.1, 0.1] and t.scale == [0.9, 1.1] and t.shear == [-5.0, 5.0]
    assert t.interpolation == "bilinear"
    t = cli.make_augment(p.parse_args(["--translate", "0.2"]), None)
    assert t.degrees == [-0.0, 0.0] and t.translate == [0.2, 0.2] and t.scale is None and t.shear is None


@pytest.mark.parametrize("flags, msg", [
    (["--rotate", "10", "--mixup", "0.2"], "--mixup cannot be combined"),
    (["--translate", "0.1", "--mixup", "0.2"], "--mixup cannot be combined"),
    (["--rotate", "-1"], "--rotate must be non-negative"),
    (["--translate", "1.5"], "--translate must lie in [0, 1]"),
    (["--scale-range", "1.1", "0.9"], "--scale-range needs 0 < LO <= HI"),
    (["--shear", "-2"], "--shear must be non-negative"),
])
def test_cli_refuses_bad_augmentation(flags, msg):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py")] + flags, capture_output=True, text=True, timeout=60,
                         cwd=ROOT)
    assert out.returncode != 0 and msg in out.stderr, out.stderr[-500:]


def test_train_script_runs_with_augmentation_on_gloo():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "2", "--backend", "gloo", "--epochs", "1",
                          "--steps", "3", "--rotate", "10", "--translate", "0.1", "--log-interval", "1", "--samples", "2000"],
                         capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-1500:] + out.stderr[-1500:]
    losses = [float(l.rsplit(" ", 1)[1]) for l in out.stdout.splitlines() if "Loss:" in l]
    assert len(losses) == 3 and all(math.isfinite(v) for v in losses), out.stdout[-1500:]


def test_resumed_run_draws_the_uninterrupted_affine_sequence(tmp_path):
    """The augmentation's generator is seeded from (epoch, rank), so a run resumed from an epoch's checkpoint trains epoch 2 on the
    images an uninterrupted run warps."""
    base = [sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "1", "--backend", "gloo", "--rotate", "15", "--translate", "0.1",
            "--steps", "3", "--samples", "400", "--log-interval", "1"]

    def run(*extra):
        out = subprocess.run(base + list(extra), capture_output=True, text=True, timeout=240, cwd=ROOT)
        assert out.returncode == 0, out.stderr[-2000:]
        return re.findall(r"Epoch \[2/2\], Step \[\d+/\d+\], Loss: \S+", out.stdout)

    ck = str(tmp_path / "run.pt")
    whole = run("--epochs", "2")
    run("--epochs", "1", "--checkpoint", ck)
    resumed = run("--epochs", "2", "--resume", ck)
    assert len(whole) == 3 and resumed == whole, (whole, resumed)
