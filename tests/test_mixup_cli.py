"""pdt.data.mixup against an explicit float64 reference, and train_mnist.py --mixup: parsed, validated, and run on the CPU."""
import math
import os
import re
import subprocess
import sys

import pytest
import torch

import pytorch_distributed_train_b200 as pdt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cli_parses_and_validates_mixup():
    from pytorch_distributed_train_b200 import cli

    p = cli.build_parser()
    assert p.parse_args([]).mixup is None
    assert p.parse_args(["--mixup", "0.2"]).mixup == 0.2
    for alpha in ("0.2", "1", "4"):
        cli.check_args(p, p.parse_args(["--mixup", alpha]))
    for alpha in ("0", "-0.5"):
        out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py"), "--mixup", alpha], capture_output=True,
                             text=True, timeout=60, cwd=ROOT)
        assert out.returncode != 0 and "--mixup must be positive" in out.stderr, (alpha, out.stderr[-500:])


def _lambda(alpha, seed):
    """torch.distributions.Beta(α, α)'s draw (torchvision MixUp's λ) under the given seed of torch's default generator."""
    state = torch.random.get_rng_state()
    try:
        torch.manual_seed(seed)
        return float(torch.distributions.Beta(torch.tensor([alpha]), torch.tensor([alpha])).sample(()))
    finally:
        torch.random.set_rng_state(state)


@pytest.mark.parametrize("alpha", [0.2, 1.0, 5.0])
def test_mixup_matches_float64_definition(alpha):
    g = torch.Generator().manual_seed(7)
    images = torch.rand(9, 1, 28, 28, generator=g)
    labels = torch.randint(0, 10, (9,), generator=g)
    labels[3] = labels[2]   # two neighbours of the same class: their target entries add up
    x0 = images.clone()
    q = pdt.data.mixup(images, labels, 10, alpha, torch.Generator().manual_seed(11))
    lam = _lambda(alpha, 11)   # the same draw from the same seed
    assert 0.0 <= lam <= 1.0
    xd = x0.double()
    onehot = torch.nn.functional.one_hot(labels, 10).double()
    ref_x = lam * xd + (1 - lam) * xd.roll(1, 0)
    ref_q = lam * onehot + (1 - lam) * onehot.roll(1, 0)
    assert q.dtype == torch.float32 and q.shape == (9, 10)
    assert torch.allclose(images.double(), ref_x, rtol=1e-6, atol=1e-7)
    assert torch.allclose(q.double(), ref_q, rtol=1e-6, atol=1e-7)
    assert torch.allclose(q.sum(1), torch.ones(9))
    # the same generator state gives the same batch
    again = x0.clone()
    assert torch.equal(pdt.data.mixup(again, labels, 10, alpha, torch.Generator().manual_seed(11)), q) and torch.equal(again, images)


def test_mixup_keeps_pinned_images_in_place():
    if not torch.cuda.is_available():
        pytest.skip("pinned memory needs CUDA")
    images = torch.rand(4, 1, 28, 28).pin_memory()
    ptr = images.data_ptr()
    pdt.data.mixup(images, torch.arange(4), 10, 0.2, torch.Generator().manual_seed(0))
    assert images.is_pinned() and images.data_ptr() == ptr


def test_mixup_rejects_non_positive_alpha():
    with pytest.raises(ValueError, match="alpha"):
        pdt.data.mixup(torch.rand(2, 1, 28, 28), torch.arange(2), 10, 0.0)


@pytest.mark.parametrize("extra", [[], ["--accumulation-steps", "2"]], ids=["k1", "k2"])
def test_train_script_runs_with_mixup(extra):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "1", "--backend", "gloo", "--mixup", "0.2",
                          "--steps", "2", "--samples", "400", "--epochs", "1", "--log-interval", "1"] + extra,
                         capture_output=True, text=True, timeout=240, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "Epoch [1/1], Step [2/" in out.stdout and "Step [3/" not in out.stdout, out.stdout[-1000:]
    losses = [float(v) for v in re.findall(r"Loss: (\S+)", out.stdout)]
    assert len(losses) == 2 and all(math.isfinite(v) for v in losses), out.stdout[-1000:]


def test_resumed_run_draws_the_uninterrupted_mixup_sequence(tmp_path):
    """The λ generator is seeded from (epoch, rank), so a run resumed from an epoch's checkpoint trains epoch 2 on the batches an
    uninterrupted run mixes."""
    base = [sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "1", "--backend", "gloo", "--mixup", "0.2", "--steps", "3",
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
