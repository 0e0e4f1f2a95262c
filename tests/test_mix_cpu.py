"""pdt.data.MixUp and pdt.data.CutMix without a GPU: the CPU path bit for bit against torchvision's transforms under one seed, a
float64 reference of the definition given the recorded (λ, r_x, r_y), torchvision's argument and call checks, and
train_mnist.py's --cutmix.

The reference (also used by test_mix.py on the GPU) forms torchvision's CutMix box from (λ, r_x, r_y) in float64,
    r = ½·√(1 − λ),  x1 = max(r_x − ⌊r·W⌋, 0),  y1 = max(r_y − ⌊r·H⌋, 0),  x2 = min(r_x + ⌊r·W⌋, W),  y2 = min(r_y + ⌊r·H⌋, H),
    λ_adj = 1 − (x2 − x1)(y2 − y1)/(W·H),
and mixes image i with image i − 1 (image 0 with image B − 1) as torchvision's fp32 tensor ops round:
    fl(fl(x[i−1]·fp32(1 − λ)) + fl(x[i]·fp32(λ))).
Each product and sum is formed in float64 and rounded to fp32; with 53 ≥ 2·24 + 2 bits that double rounding equals the fp32
operation's rounding, so the reference is exact, not a tolerance."""
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

try:
    from torchvision.transforms import v2 as TV2
except Exception:   # noqa: BLE001  (torchvision is optional)
    TV2 = None


# ---- the float64 reference --------------------------------------------------------------------------------------------------

def cutmix_box(lam, r_x, r_y, H, W):
    """torchvision's CutMix.make_params from (λ, r_x, r_y): ((x1, y1, x2, y2), λ_adj)."""
    r = 0.5 * math.sqrt(1.0 - lam)
    r_w_half, r_h_half = int(r * W), int(r * H)
    x1, y1 = max(int(r_x) - r_w_half, 0), max(int(r_y) - r_h_half, 0)
    x2, y2 = min(int(r_x) + r_w_half, W), min(int(r_y) + r_h_half, H)
    return (x1, y1, x2, y2), 1.0 - (x2 - x1) * (y2 - y1) / (W * H)


def _f32(a):
    return a.astype(np.float32).astype(np.float64)


def blend(a, lam):
    """Rows of a (float64 holding fp32 values) mixed with their roll-by-one partners, rounded as torchvision's fp32 ops round."""
    partner = np.roll(a, 1, axis=0)
    return _f32(_f32(partner * np.float64(np.float32(1.0 - lam))) + _f32(a * np.float64(np.float32(lam)))).astype(np.float32)


def reference_mix(x, labels, num_classes, record, cutmix):
    """(images, targets) the definition gives for the recorded parameters; `record` is (λ) or (λ, r_x, r_y, x1, y1, x2, y2, λ_adj).
    Index labels outside [0, num_classes) give rows without mass."""
    x = x.detach().cpu().double().numpy()
    labels = labels.detach().cpu()
    rec = [float(v) for v in record.detach().cpu().double()]
    if labels.ndim == 1:
        lab = labels.numpy()
        t = np.zeros((len(lab), num_classes))
        ok = (lab >= 0) & (lab < num_classes)
        t[np.nonzero(ok)[0], lab[ok]] = 1.0
    else:
        t = labels.double().numpy()
    lam = rec[0]
    if not cutmix:
        return torch.from_numpy(blend(x, lam)), torch.from_numpy(blend(t, lam))
    H, W = x.shape[-2:]
    (x1, y1, x2, y2), lam_adj = cutmix_box(lam, rec[1], rec[2], H, W)
    assert (x1, y1, x2, y2) == tuple(int(v) for v in rec[3:7]) and lam_adj == rec[7], (rec, (x1, y1, x2, y2), lam_adj)
    out = x.copy()
    out[..., y1:y2, x1:x2] = np.roll(x, 1, axis=0)[..., y1:y2, x1:x2]
    return torch.from_numpy(out.astype(np.float32)), torch.from_numpy(blend(t, lam_adj))


def check_against_reference(x, labels, num_classes, out, targets, record, cutmix):
    want_x, want_t = reference_mix(x, labels, num_classes, record, cutmix)
    assert torch.equal(out.cpu(), want_x)
    assert torch.equal(targets.cpu(), want_t)


def _labels(B, prob, seed=0, K=10):
    g = torch.Generator().manual_seed(seed)
    return torch.softmax(torch.randn(B, K, generator=g), 1) if prob else torch.randint(0, K, (B,), generator=g)


# ---- against torchvision ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cutmix", [False, True])
@pytest.mark.parametrize("alpha", [0.2, 1.0, 5.0])
@pytest.mark.parametrize("shape", [(9, 1, 28, 28), (7, 3, 16, 20), (1, 1, 28, 28)])
@pytest.mark.parametrize("prob", [False, True])
def test_cpu_matches_torchvision_bit_for_bit(cutmix, alpha, shape, prob):
    if TV2 is None:
        pytest.skip("torchvision is not importable")
    x = torch.rand(shape, generator=torch.Generator().manual_seed(1))
    y = _labels(shape[0], prob)
    ours = (pdt.data.CutMix if cutmix else pdt.data.MixUp)(alpha=alpha, num_classes=10)
    theirs = (TV2.CutMix if cutmix else TV2.MixUp)(alpha=alpha, num_classes=10)
    for seed in (0, 1, 2):
        torch.manual_seed(seed)
        a, ta = ours(x, y)
        torch.manual_seed(seed)
        b, tb = theirs(x, y)
        assert torch.equal(a, b) and torch.equal(ta, tb), seed
        assert ta.dtype == torch.float32 and ta.shape == (shape[0], 10)
    # an own generator draws what torch's default one draws from the same seed
    torch.manual_seed(7)
    b, tb = theirs(x, y)
    ours.generator = torch.Generator().manual_seed(7)
    a, ta = ours(x, y)
    assert torch.equal(a, b) and torch.equal(ta, tb)


# ---- the float64 reference --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cutmix", [False, True])
@pytest.mark.parametrize("shape", [(9, 1, 28, 28), (7, 3, 16, 20), (1, 1, 5, 3)])
@pytest.mark.parametrize("prob", [False, True])
def test_cpu_matches_float64_reference(cutmix, shape, prob):
    x = torch.rand(shape, generator=torch.Generator().manual_seed(2))
    y = _labels(shape[0], prob, seed=3)
    t = (pdt.data.CutMix if cutmix else pdt.data.MixUp)(alpha=0.7, num_classes=10, generator=torch.Generator().manual_seed(4),
                                                          record_params=True)
    for _ in range(20):
        out, targets = t(x, y)
        rec = t.last_params
        assert rec.dtype == torch.float64 and rec.shape == ((8,) if cutmix else (1,))
        check_against_reference(x, y, 10, out, targets, rec, cutmix)
    assert torch.equal(x, torch.rand(shape, generator=torch.Generator().manual_seed(2)))   # the input is not touched


def test_reference_box_follows_torchvision_formula():
    # hand-checked boxes: λ = 0.75 → r = 0.25, ⌊r·28⌋ = 7; clamped at both edges; λ = 1 → an empty box
    assert cutmix_box(0.75, 10, 20, 28, 28) == ((3, 13, 17, 27), 1.0 - 14 * 14 / 784)
    assert cutmix_box(0.75, 0, 27, 28, 28) == ((0, 20, 7, 28), 1.0 - 7 * 8 / 784)
    assert cutmix_box(1.0, 5, 5, 16, 20) == ((5, 5, 5, 5), 1.0)
    assert cutmix_box(0.0, 10, 8, 16, 20) == ((0, 0, 20, 16), 0.0)


def test_mixup_function_unchanged_by_the_shared_arithmetic():
    """pdt.data.mixup (the --mixup path) and MixUp share their arithmetic and their λ: the same draw gives the same batch."""
    x = torch.rand(12, 1, 28, 28, generator=torch.Generator().manual_seed(5))
    y = _labels(12, False, seed=6)
    a = x.clone()
    ta = pdt.data.mixup(a, y, 10, 0.4, torch.Generator().manual_seed(8))
    b, tb = pdt.data.MixUp(alpha=0.4, num_classes=10, generator=torch.Generator().manual_seed(8))(x, y)
    assert torch.equal(a, b) and torch.equal(ta, tb)


# ---- checks -----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cls", ["MixUp", "CutMix"])
def test_constructor_and_call_checks(cls):
    T = getattr(pdt.data, cls)
    for alpha in (0.0, -1.0, float("nan")):
        with pytest.raises(ValueError):
            T(alpha=alpha, num_classes=10)
    with pytest.raises(TypeError):
        T(alpha=1.0, num_classes=10, labels_getter="default")   # not supported
    with pytest.raises(TypeError):
        T(1.0)   # keyword-only, as torchvision's
    t = T(num_classes=10)
    x, y = torch.rand(4, 1, 8, 8), torch.randint(0, 10, (4,))
    # (arguments, error, message, torchvision raises the same): a list of labels meets torchvision's labels_getter first
    cases = [
        ((x, [1, 2, 3, 4]), ValueError, "The labels must be a tensor", False),
        ((x, y.view(2, 2, 1)), ValueError, "labels should be index based with shape (batch_size,)", True),
        ((x, torch.rand(4, 5)), ValueError, "the number of elements in last dimension must match num_classes: 5 != 10", True),
        ((x[0], y), ValueError, "Expected a batched input with 4 dims, but got 3 dimensions instead.", True),
        ((x[:3], y), ValueError, "does not match the batch size of the labels: 3 != 4.", True),
        ((x.double(), y), TypeError, "images must be float32", False),
        ((x, y.int()), TypeError, "index labels must be torch.int64", False),
        ((x, torch.rand(4, 10).double()), TypeError, "probability labels must be torch.float32", False),
    ]
    for args, err, msg, same in cases:
        with pytest.raises(err, match=re.escape(msg)):
            t(*args)
        if TV2 is not None and same:
            with pytest.raises(err, match=re.escape(msg)):
                getattr(TV2, cls)(num_classes=10)(*args)
    with pytest.raises(ValueError, match=re.escape("num_classes must be passed if the labels are index-based (1D)")):
        T()(x, y)
    out, targets = T()(x, torch.rand(4, 6))   # probability labels need no num_classes
    assert targets.shape == (4, 6)


def test_empty_batch():
    for T in (pdt.data.MixUp, pdt.data.CutMix):
        out, targets = T(num_classes=10)(torch.zeros(0, 1, 28, 28), torch.zeros(0, dtype=torch.int64))
        assert out.shape == (0, 1, 28, 28) and targets.shape == (0, 10)


# ---- the CLI ----------------------------------------------------------------------------------------------------------------

def test_cli_parses_and_validates_cutmix():
    p = cli.build_parser()
    assert p.parse_args([]).cutmix is None
    a = p.parse_args(["--cutmix", "0.5", "--rotate", "10", "--accumulation-steps", "2", "--label-smoothing", "0.1", "--ema-decay", "0.9",
                      "--eval"])
    cli.check_args(p, a)
    assert a.cutmix == 0.5


@pytest.mark.parametrize("flags, msg", [
    (["--cutmix", "1.0", "--mixup", "0.2"], "--cutmix cannot be combined with --mixup"),
    (["--cutmix", "0"], "--cutmix must be positive"),
    (["--cutmix", "-1"], "--cutmix must be positive"),
])
def test_cli_refuses_bad_cutmix(flags, msg):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py")] + flags, capture_output=True, text=True, timeout=60,
                         cwd=ROOT)
    assert out.returncode != 0 and msg in out.stderr, out.stderr[-500:]


@pytest.mark.parametrize("extra", [[], ["--accumulation-steps", "2"], ["--rotate", "10"]])
def test_train_script_runs_with_cutmix_on_gloo(extra):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "1", "--backend", "gloo", "--cutmix", "1.0",
                          "--epochs", "1", "--steps", "3", "--log-interval", "1", "--samples", "1000"] + extra,
                         capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-1500:] + out.stderr[-1500:]
    losses = [float(v) for v in re.findall(r"Step \[\d+/\d+\], Loss: (\S+)", out.stdout)]
    assert len(losses) == 3 and all(math.isfinite(v) for v in losses), out.stdout[-1500:]


def test_resumed_run_draws_the_uninterrupted_cutmix_sequence(tmp_path):
    """CutMix's generator is seeded from (epoch, rank), so a run resumed from an epoch's checkpoint mixes epoch 2 as an
    uninterrupted run does."""
    base = [sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "1", "--backend", "gloo", "--cutmix", "1.0", "--steps", "3",
            "--samples", "400", "--log-interval", "1"]

    def run(*extra):
        out = subprocess.run(base + list(extra), capture_output=True, text=True, timeout=240, cwd=ROOT)
        assert out.returncode == 0, out.stderr[-2000:]
        return re.findall(r"Epoch \[2/2\], Step \[\d+/\d+\], Loss: \S+", out.stdout)

    ck = str(tmp_path / "run.pt")
    whole = run("--epochs", "2")
    run("--epochs", "1", "--checkpoint", ck)
    resumed = run("--epochs", "2", "--resume", ck)
    assert len(whole) == 3 and resumed == whole, (whole, resumed)
