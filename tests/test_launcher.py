"""Launcher contract (ref: ddp_example.py:111; spawn.py:79-96,145-211)."""
import os
import signal
import time

import pytest

from pytorch_distributed_train_b200 import launcher


def _ok(i, tmp):
    with open(os.path.join(tmp, f"{i}.txt"), "w") as f:
        f.write(f"{i} {os.environ.get('PDT_LOCAL_RANK')} {os.environ.get('PDT_LOCAL_WORLD_SIZE')}")


def _raiser(i):
    if i == 1:
        raise ValueError("boom from child one")
    time.sleep(30)


def _killed(i):
    if i == 0:
        os.kill(os.getpid(), signal.SIGKILL)
    time.sleep(30)


def _exit3(i):
    if i == 0:
        os._exit(3)
    time.sleep(30)


def test_spawn_runs_every_rank(tmp_path):
    launcher.spawn(_ok, args=(str(tmp_path),), nprocs=3)
    got = sorted(open(tmp_path / f"{i}.txt").read() for i in range(3))
    assert got == ["0 0 3", "1 1 3", "2 2 3"]


def test_child_exception_reaches_parent_and_siblings_die():
    t0 = time.time()
    with pytest.raises(launcher.ProcessRaisedException) as ei:
        launcher.spawn(_raiser, nprocs=2, grace_period=2.0)
    assert "boom from child one" in str(ei.value) and "ValueError" in str(ei.value)
    assert ei.value.error_index == 1
    assert time.time() - t0 < 20, "siblings must be terminated, not waited for"


def test_child_killed_by_signal():
    with pytest.raises(launcher.ProcessExitedException) as ei:
        launcher.spawn(_killed, nprocs=2, grace_period=2.0)
    assert ei.value.signal_name == "SIGKILL" and ei.value.error_index == 0


def test_child_exit_code():
    with pytest.raises(launcher.ProcessExitedException) as ei:
        launcher.spawn(_exit3, nprocs=2, grace_period=2.0)
    assert ei.value.exit_code == 3


def test_nonblocking_join_context(tmp_path):
    ctx = launcher.start_processes(_ok, args=(str(tmp_path),), nprocs=2, join=False)
    assert len(ctx.pids()) == 2
    while not ctx.join():
        pass
    ctx.cleanup()


def test_only_spawn_start_method():
    with pytest.raises(ValueError):
        launcher.spawn(_ok, nprocs=1, start_method="fork")


def test_script_launcher_env_rendezvous(tmp_path):
    """`python -m pytorch_distributed_train_b200.launcher --nproc-per-node 2 script.py` — the torchrun-style entry."""
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "job.py"
    script.write_text(
        "import os, sys, torch\n"
        f"sys.path.insert(0, {root!r})\n"
        "import pytorch_distributed_train_b200 as pdt\n"
        "pdt.init_process_group('gloo', init_method='env://')\n"
        "t = torch.tensor([float(pdt.get_rank() + 1)])\n"
        "pdt.distributed.all_reduce(t)\n"
        "print(f\"rank {os.environ['RANK']}/{os.environ['WORLD_SIZE']} local {os.environ['LOCAL_RANK']} sum {t.item()} arg {sys.argv[1]}\", flush=True)\n"
        "pdt.destroy_process_group()\n"
        "sys.exit(0)\n")
    out = subprocess.run([sys.executable, "-m", "pytorch_distributed_train_b200.launcher", "--nproc-per-node", "2", str(script), "hello"],
                         capture_output=True, text=True, timeout=120, cwd=root)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "rank 0/2 local 0 sum 3.0 arg hello" in out.stdout and "rank 1/2 local 1 sum 3.0 arg hello" in out.stdout
    bad = tmp_path / "bad.py"
    bad.write_text("import os\nif os.environ['RANK'] == '1':\n    raise ValueError('boom on rank 1')\nimport time; time.sleep(30)\n")
    out = subprocess.run([sys.executable, "-m", "pytorch_distributed_train_b200.launcher", "--nproc-per-node", "2", str(bad)],
                         capture_output=True, text=True, timeout=120, cwd=root)
    assert out.returncode == 1 and "boom on rank 1" in out.stderr   # sibling killed, traceback surfaced, bounded time
