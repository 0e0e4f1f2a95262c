"""train_mnist.py --label-smoothing: parsed, validated, and passed to the criterion of a run."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cli_parses_and_validates_label_smoothing():
    from pytorch_distributed_train_b200 import cli

    p = cli.build_parser()
    assert p.parse_args([]).label_smoothing == 0.0
    assert p.parse_args(["--label-smoothing", "0.1"]).label_smoothing == 0.1
    for eps in ("0", "0.1", "1"):
        cli.check_args(p, p.parse_args(["--label-smoothing", eps]))
    for eps in ("-0.1", "1.5"):
        out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py"), "--label-smoothing", eps], capture_output=True,
                             text=True, timeout=60, cwd=ROOT)
        assert out.returncode != 0 and "--label-smoothing must lie in [0, 1]" in out.stderr, (eps, out.stderr[-500:])


def test_train_script_runs_with_label_smoothing():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "1", "--backend", "gloo", "--label-smoothing", "0.1",
                          "--steps", "2", "--samples", "400", "--epochs", "1", "--log-interval", "1"],
                         capture_output=True, text=True, timeout=240, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "Epoch [1/1], Step [2/" in out.stdout and "Step [3/" not in out.stdout, out.stdout[-1000:]
