"""Auxiliary subsystems on the CPU box: watchdog, rank-aware logging, NVTX no-op,
clock sampler fallback, device-timer helpers that must degrade gracefully without a GPU."""
import json
import os
import time

import torch

import pytorch_distributed_train_b200 as pdt
from mp_helpers import free_port


def _watchdog_entry(rank, world, init, outdir):
    pdt.init_process_group("gloo", init_method=init, world_size=world, rank=rank, timeout=30.0)
    wd = pdt.utils.Watchdog(interval=0.2, timeout=1.0, abort=False).start()
    if rank == 1:
        time.sleep(1.0)      # a few heartbeats, then die without saying goodbye
        os._exit(0)
    t0 = time.time()
    while not wd.dead_peers and time.time() - t0 < 15:
        time.sleep(0.1)
    with open(os.path.join(outdir, "r0.json"), "w") as f:
        json.dump({"dead": wd.dead_peers, "seconds": time.time() - t0}, f)
        f.flush()
    os._exit(0)              # peers are gone: skip the orderly teardown


def test_watchdog_notices_a_silent_peer(tmp_path):
    pdt.spawn(_watchdog_entry, args=(2, f"tcp://127.0.0.1:{free_port()}", str(tmp_path)), nprocs=2, grace_period=5.0)
    res = json.load(open(tmp_path / "r0.json"))
    assert res["dead"] == [1] and res["seconds"] < 10, res


def test_rank_zero_print_and_logger(capsys):
    pdt.utils.rank_zero_print("hello", 3)       # no process group: behaves like print
    assert capsys.readouterr().out == "hello 3\n"
    log = pdt.utils.get_logger("pdt.test")
    log.setLevel("INFO")
    log.info("message %d", 7)
    err = capsys.readouterr().err
    assert "[pdt][rank" in err and "INFO message 7" in err


def test_nvtx_and_clock_sampler_degrade_without_a_gpu():
    with pdt.utils.nvtx_range("phase"):
        x = torch.ones(3).sum().item()
    assert x == 3
    with pdt.utils.ClockSampler(0) as c:
        time.sleep(0.02)
    s = c.summary()
    assert set(s) >= {"sm_mhz", "sm_max_mhz", "reasons", "samples"}
    if not torch.cuda.is_available():
        assert s["samples"] == 0 and s["sm_mhz"] is None


def test_upcoming_targets_and_rider_contexts_nest_and_restore():
    """Engine-level announcements (ops.functional): nested contexts restore the outer state; nothing leaks after exit."""
    import torch

    from pytorch_distributed_train_b200.ops import functional as OF

    a, b = torch.zeros(3, dtype=torch.int64), torch.ones(3, dtype=torch.int64)
    assert OF._upcoming_target is None and OF._loss_read_after_backward is False and OF._sgd_rider_enabled is False
    with OF.upcoming_targets(a, loss_read_after_backward=True):
        assert OF._upcoming_target is a and OF._loss_read_after_backward is True
        with OF.upcoming_targets(b):
            assert OF._upcoming_target is b and OF._loss_read_after_backward is False
        assert OF._upcoming_target is a and OF._loss_read_after_backward is True
        with OF.sgd_rider_enabled():
            assert OF._sgd_rider_enabled is True
        assert OF._sgd_rider_enabled is False
    assert OF._upcoming_target is None and OF._loss_read_after_backward is False


def test_sgd_rider_only_arms_for_the_fused_cuda_convnet():
    """optim.SGD.ride_on_backward refuses everything but a CUDA fp32 reference ConvNet whose parameters are exactly the optimizer's."""
    import torch

    import pytorch_distributed_train_b200 as pdt
    from pytorch_distributed_train_b200.ops import functional as OF

    net = pdt.models.ConvNet()
    opt = pdt.optim.SGD(net.parameters(), 0.1)
    assert opt.ride_on_backward(net) is False            # CPU parameters
    assert opt.ride_on_backward(torch.nn.Linear(4, 4)) is False   # not the ConvNet
    part = pdt.optim.SGD(list(net.parameters())[:4], 0.1)
    assert part.ride_on_backward(net) is False           # optimizer does not own every parameter
    assert OF._sgd_rider is None
    opt.step()                                           # the ordinary path still runs (no gradients: a no-op)
