"""Weight averaging: pdt.optim.swa_utils.AveragedModel against torch's on the CPU (torch's path) and on the GPU (the native
avg_multi kernel), GraphedTrainStep(averaged_model=...), checkpoints and train_mnist.py --ema-decay."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F
from torch.optim import swa_utils as tsw

import pytorch_distributed_train_b200 as pdt
from pytorch_distributed_train_b200.optim import swa_utils as psw

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Net(torch.nn.Module):
    """Parameters and buffers of every kind AveragedModel sees: fp32 weights, BatchNorm running statistics, int64
    num_batches_tracked."""

    def __init__(self, width=7):
        super().__init__()
        self.lin = torch.nn.Linear(5, width)
        self.bn = torch.nn.BatchNorm1d(width)
        self.out = torch.nn.Linear(width, 3)

    def forward(self, x):
        return self.out(self.bn(self.lin(x)))


def _perturb(model, seed):
    """One 'training step': new weights and buffers, as after optimizer.step() and a forward in training mode."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in model.parameters():
            p.add_(torch.randn(p.shape, generator=g).to(p.device) * 0.1)
        for b in model.buffers():
            if b.dtype == torch.int64:
                b.add_(int(torch.randint(1, 4, (), generator=g)))
            else:
                b.mul_(0.9).add_(torch.rand(b.shape, generator=g).to(b.device))


def _avg_fns():
    return {
        "ema0.9": (dict(multi_avg_fn=psw.get_ema_multi_avg_fn(0.9)), dict(multi_avg_fn=tsw.get_ema_multi_avg_fn(0.9))),
        "swa": (dict(multi_avg_fn=psw.get_swa_multi_avg_fn()), dict(multi_avg_fn=tsw.get_swa_multi_avg_fn())),
        "default": (dict(), dict()),
        "custom": (dict(avg_fn=lambda a, p, n: 0.25 * a + 0.75 * p), dict(avg_fn=lambda a, p, n: 0.25 * a + 0.75 * p)),
    }


def _states_equal(a, b):
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb)
    for k in sa:
        assert sa[k].dtype == sb[k].dtype and torch.equal(sa[k].cpu(), sb[k].cpu()), k


# =====================================================================================================================
# CPU: torch's path, bit for bit
# =====================================================================================================================
@pytest.mark.parametrize("fn", ["ema0.9", "swa", "default", "custom"])
@pytest.mark.parametrize("use_buffers", [False, True])
def test_cpu_matches_torch_bit_for_bit(fn, use_buffers):
    torch.manual_seed(0)
    model = _Net()
    ours_kw, theirs_kw = _avg_fns()[fn]
    ours = psw.AveragedModel(model, use_buffers=use_buffers, **ours_kw)
    theirs = tsw.AveragedModel(model, use_buffers=use_buffers, **theirs_kw)
    assert isinstance(ours, tsw.AveragedModel)
    for i in range(5):
        _perturb(model, i)
        if use_buffers and fn == "swa" and i > 0:
            # torch's swa_update cannot average the int64 num_batches_tracked: the same error from both (the default takes the
            # per-tensor get_swa_avg_fn on the CPU, which can)
            with pytest.raises(RuntimeError) as e1:
                ours.update_parameters(model)
            with pytest.raises(RuntimeError) as e2:
                theirs.update_parameters(model)
            assert str(e1.value) == str(e2.value)
            return
        ours.update_parameters(model)
        theirs.update_parameters(model)
        _states_equal(ours, theirs)
    assert ours.n_averaged.item() == 5


def test_state_dicts_load_both_ways():
    torch.manual_seed(1)
    model = _Net()
    ours = psw.AveragedModel(model, multi_avg_fn=psw.get_ema_multi_avg_fn(0.5), use_buffers=True)
    for i in range(3):
        _perturb(model, i)
        ours.update_parameters(model)
    theirs = tsw.AveragedModel(_Net(), multi_avg_fn=tsw.get_ema_multi_avg_fn(0.5), use_buffers=True)
    theirs.load_state_dict(ours.state_dict())
    _states_equal(ours, theirs)
    _perturb(model, 9)
    theirs.update_parameters(model)
    back = psw.AveragedModel(_Net(), multi_avg_fn=psw.get_ema_multi_avg_fn(0.5), use_buffers=True)
    back.load_state_dict(theirs.state_dict())
    _states_equal(back, theirs)
    assert back.n_averaged.item() == 4


@pytest.mark.parametrize("decay", [-0.1, 1.5])
def test_decay_is_validated_as_torch_does(decay):
    with pytest.raises(ValueError) as ours:
        psw.get_ema_multi_avg_fn(decay)
    with pytest.raises(ValueError) as theirs:
        tsw.get_ema_multi_avg_fn(decay)
    assert str(ours.value) == str(theirs.value)


def test_torch_names_are_reexported():
    assert pdt.optim.swa_utils is psw
    assert psw.SWALR is tsw.SWALR and psw.update_bn is tsw.update_bn
    assert psw.get_ema_avg_fn is tsw.get_ema_avg_fn and psw.get_swa_avg_fn is tsw.get_swa_avg_fn


def test_cpu_model_has_no_native_plan():
    ours = psw.AveragedModel(_Net(), multi_avg_fn=psw.get_ema_multi_avg_fn(0.9))
    assert isinstance(ours.native_plan(_Net()), str)


@pytest.mark.parametrize("bad", ["-0.5", "1.01"])
def test_cli_rejects_ema_decay_outside_unit_interval(bad):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py"), "--ema-decay", bad],
                         capture_output=True, text=True, timeout=60, cwd=ROOT)
    assert out.returncode != 0 and "--ema-decay must lie in [0, 1]" in out.stderr
    from pytorch_distributed_train_b200 import cli

    assert cli.build_parser().parse_args([]).ema_decay is None


def _torch_ddp_ema(rank, world, port, steps, lr, decay):
    """torch DDP + gloo + torch's AveragedModel (EMA of weights and buffers) on train_mnist.py's data, model and seed."""
    import torch.distributed as td

    from pytorch_distributed_train_b200 import data as pdata

    td.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", world_size=world, rank=rank)
    try:
        torch.manual_seed(0)
        model = pdt.models.ConvNet()
        ema = tsw.AveragedModel(model, multi_avg_fn=tsw.get_ema_multi_avg_fn(decay), use_buffers=True)
        ddp = torch.nn.parallel.DistributedDataParallel(model)
        opt = torch.optim.SGD(ddp.parameters(), lr)
        crit = torch.nn.CrossEntropyLoss()
        ds = pdata.SyntheticMNIST(600, seed=0, num_classes=10, image_shape=(1, 28, 28))
        loader = torch.utils.data.DataLoader(ds, batch_size=100, shuffle=False,
                                             sampler=torch.utils.data.DistributedSampler(ds, num_replicas=world, rank=rank))
        for i, (x, y) in enumerate(loader):
            if i >= steps:
                break
            loss = crit(ddp(x), y)
            opt.zero_grad()
            loss.backward()
            opt.step()
            ema.update_parameters(model)
        return {k: v.clone() for k, v in ema.state_dict().items()}
    finally:
        td.destroy_process_group()


def test_train_script_ema_matches_torch_ddp_gloo(tmp_path):
    from mp_helpers import free_port, run_ranks

    ck = str(tmp_path / "ema.pt")
    cmd = [sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "2", "--backend", "gloo", "--lr", "0.1", "--ema-decay", "0.9",
           "--steps", "3", "--samples", "600", "--epochs", "1", "--log-interval", "3", "--checkpoint", ck]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=240, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    payload = torch.load(ck, map_location="cpu", weights_only=False)
    ours, model = payload["averaged_model"], payload["model"]
    ref = run_ranks(_torch_ddp_ema, 2, free_port(), 3, 0.1, 0.9)[0]
    assert list(ours) == list(ref)
    assert ours["n_averaged"].item() == 3
    for k in ref:
        assert torch.allclose(ours[k].float(), ref[k].float(), atol=1e-5, rtol=1e-4), (k, (ours[k].float() - ref[k].float()).abs().max())
    # the average lags the model: it is not a copy of it
    assert not torch.equal(ours["module.fc.weight"], model["module.fc.weight"])


# =====================================================================================================================
# GPU
# =====================================================================================================================
def _dev():
    return torch.device("cuda", 0)


class _Wide(torch.nn.Module):
    """More tensors than one table holds (48), with odd and empty sizes, plus two BatchNorms (int64 buffers)."""

    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(5)
        sizes = [0, 1, 3, 1000003] + [int(s) for s in torch.randint(1, 3000, (52,), generator=g)]
        self.ps = torch.nn.ParameterList([torch.nn.Parameter(torch.randn(s, generator=g)) for s in sizes])
        self.bn1 = torch.nn.BatchNorm1d(13)
        self.bn2 = torch.nn.BatchNorm1d(5)


def _wide_pair(decay, use_buffers):
    torch.manual_seed(0)
    model = _Wide().to(_dev())
    fn_ours = psw.get_swa_multi_avg_fn() if decay is None else psw.get_ema_multi_avg_fn(decay)
    fn_theirs = tsw.get_swa_multi_avg_fn() if decay is None else tsw.get_ema_multi_avg_fn(decay)
    ours = psw.AveragedModel(model, multi_avg_fn=fn_ours, use_buffers=use_buffers)
    theirs = tsw.AveragedModel(model, device=_dev(), multi_avg_fn=fn_theirs, use_buffers=use_buffers)
    return model, ours, theirs


def _float64_recurrence(history, decay):
    """The average of the model states in `history`, in float64."""
    avg = None
    for n, state in enumerate(history):
        if avg is None:
            avg = [t.double() for t in state]
            continue
        w = 1.0 / (n + 1) if decay is None else 1.0 - decay
        avg = [a + w * (t.double() - a) for a, t in zip(avg, state)]
    return avg


@pytest.mark.gpu
@pytest.mark.parametrize("decay", [0.0, 0.3, 0.999, 1.0, None])
@pytest.mark.parametrize("use_buffers", [False, True])
def test_native_update_matches_torch_bit_for_bit(decay, use_buffers):
    model, ours, theirs = _wide_pair(decay, use_buffers)
    plan = ours.native_plan(model)
    if decay is None and use_buffers:
        assert isinstance(plan, str) and "integer" in plan   # torch raises on the second update: not native
        return
    assert not isinstance(plan, str), plan
    assert ours.n_averaged.device == _dev()
    history = []
    for i in range(10):
        _perturb(model, i)
        history.append([p.detach().clone() for p in model.parameters()])
        ours.update_parameters(model)
        theirs.update_parameters(model)
        _states_equal(ours, theirs)
    assert ours.n_averaged.item() == 10
    ref = _float64_recurrence(history, decay)
    for a, r in zip(ours.module.parameters(), ref):
        if r.numel():
            assert (a.double() - r).abs().max().item() <= 1e-5 * max(1.0, r.abs().max().item())


@pytest.mark.gpu
def test_native_update_does_not_synchronise():
    model, ours, _ = _wide_pair(0.9, True)
    ours.update_parameters(model)   # first use allocates the reduction scratch
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for i in range(3):
            ours.update_parameters(model)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert ours.n_averaged.item() == 4


@pytest.mark.gpu
@pytest.mark.parametrize("decay", [0.7, None])
def test_captured_update_replayed_equals_eager_calls(decay):
    model, ours, _ = _wide_pair(decay, False)
    twin = psw.AveragedModel(model, multi_avg_fn=ours.multi_avg_fn)
    _perturb(model, 0)
    ours.update_parameters(model)
    twin.update_parameters(model)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        ours.update_parameters(model)
    for i in range(1, 6):
        _perturb(model, i)
        g.replay()
        twin.update_parameters(model)
    torch.cuda.synchronize()
    _states_equal(ours, twin)
    assert ours.n_averaged.item() == 6


@pytest.mark.gpu
def test_graphed_step_refuses_a_non_native_averaged_model():
    from mp_helpers import free_port

    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    torch.cuda.set_device(0)
    pdt.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{free_port()}", world_size=1, rank=0)
    try:
        model = pdt.models.ConvNet().to(_dev())
        ddp = pdt.DistributedDataParallel(model, device_ids=[0])
        x, t = torch.rand(100, 1, 28, 28, device=_dev()), torch.randint(0, 10, (100,), device=_dev())
        for avg in (tsw.AveragedModel(model, device=_dev(), multi_avg_fn=tsw.get_ema_multi_avg_fn(0.9)),
                    psw.AveragedModel(model, multi_avg_fn=tsw.get_ema_multi_avg_fn(0.9)),
                    psw.AveragedModel(model, avg_fn=tsw.get_ema_avg_fn(0.9))):
            with pytest.raises(ValueError, match="cannot be captured"):
                GraphedTrainStep(ddp, pdt.nn.CrossEntropyLoss(),
                                 pdt.optim.SGD(model.parameters(), 0.1), (x, t), averaged_model=avg)
    finally:
        pdt.destroy_process_group()


def _make_opt(kind, params):
    if kind == "sgd":
        return pdt.optim.SGD(params, 0.05)
    if kind == "sgd_momentum":
        return pdt.optim.SGD(params, 0.05, momentum=0.9)
    if kind == "adam":
        return pdt.optim.Adam(params, 1e-3)
    return pdt.optim.AdamW(params, 1e-3)


def _graphed_run(kind, max_norm, k, average, replays=6, decay=0.75, use_buffers=True):
    """(model state, averaged model state or torch's average over the replays, kernels per replay).  decay None: SWA."""
    from mp_helpers import free_port

    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    torch.cuda.set_device(0)
    pdt.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{free_port()}", world_size=1, rank=0)
    try:
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(_dev())
        lib = psw if average else tsw
        fn = lib.get_swa_multi_avg_fn() if decay is None else lib.get_ema_multi_avg_fn(decay)
        avg = (psw.AveragedModel(model, multi_avg_fn=fn, use_buffers=use_buffers) if average else
               tsw.AveragedModel(model, device=_dev(), multi_avg_fn=fn, use_buffers=use_buffers))
        opt = _make_opt(kind, model.parameters())
        g = torch.Generator(device=_dev()).manual_seed(9)
        xs = torch.rand(4, 100 * k, 1, 28, 28, device=_dev(), generator=g)
        ts = torch.randint(0, 10, (4, 100 * k), device=_dev(), generator=g)
        step = GraphedTrainStep(pdt.DistributedDataParallel(model, device_ids=[0]), pdt.nn.CrossEntropyLoss(), opt, (xs[0], ts[0]),
                                warmup=2, max_grad_norm=max_norm, accumulation_steps=k, averaged_model=avg if average else None)
        for i in range(replays):
            step(xs[i % 4], ts[i % 4], inputs_ready=True)
            if not average:
                avg.update_parameters(model)   # torch's update after each replay
        torch.cuda.synchronize()
        return ({n: v.clone() for n, v in model.state_dict().items()}, {n: v.clone() for n, v in avg.state_dict().items()},
                step.kernels_per_replay)
    finally:
        pdt.destroy_process_group()


def _assert_same(a, b):
    assert list(a) == list(b)
    for n in a:
        assert torch.equal(a[n], b[n]), (n, (a[n].double() - b[n].double()).abs().max().item())


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sgd", "sgd_momentum", "adam", "adamw"])
@pytest.mark.parametrize("max_norm", [None, 0.5])
@pytest.mark.parametrize("k", [1, 2])
@pytest.mark.parametrize("rider", ["1", "0"])
def test_graphed_step_averages_after_every_replay(kind, max_norm, k, rider, monkeypatch):
    """The model trains bit-identically with and without averaging, the averaged model equals torch's update after each replay,
    and averaging costs one launch per replay."""
    monkeypatch.setenv("PDT_SGD_RIDER", rider)
    plain_model, torch_avg, plain_kernels = _graphed_run(kind, max_norm, k, average=False)
    model, avg, kernels = _graphed_run(kind, max_norm, k, average=True)
    _assert_same(model, plain_model)
    _assert_same(avg, torch_avg)
    assert avg["n_averaged"].item() == 6
    assert kernels == plain_kernels + 1, (kernels, plain_kernels)
    if rider == "1":
        assert plain_kernels == 3 * k


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sgd_momentum", "adamw"])
@pytest.mark.parametrize("max_norm", [None, 0.5])
@pytest.mark.parametrize("decay", [0.3, None])
def test_graphed_step_copies_buffers_and_averages_swa(kind, max_norm, decay):
    """use_buffers=False (the buffers are copied) under EMA with the w >= 0.5 branch of lerp, and under SWA."""
    plain_model, torch_avg, plain_kernels = _graphed_run(kind, max_norm, 1, average=False, decay=decay, use_buffers=False)
    model, avg, kernels = _graphed_run(kind, max_norm, 1, average=True, decay=decay, use_buffers=False)
    _assert_same(model, plain_model)
    _assert_same(avg, torch_avg)
    assert kernels == plain_kernels + 1 == 4, (kernels, plain_kernels)


class _TorchConvNet(torch.nn.Module):
    """The ConvNet's modules under the same names, run by torch alone."""

    def __init__(self):
        super().__init__()
        self.layer1 = torch.nn.Sequential(torch.nn.Conv2d(1, 16, 5, 1, 2), torch.nn.BatchNorm2d(16), torch.nn.ReLU(), torch.nn.MaxPool2d(2, 2))
        self.layer2 = torch.nn.Sequential(torch.nn.Conv2d(16, 32, 5, 1, 2), torch.nn.BatchNorm2d(32), torch.nn.ReLU(), torch.nn.MaxPool2d(2, 2))
        self.fc = torch.nn.Linear(7 * 7 * 32, 10)

    def forward(self, x):
        return self.fc(self.layer2(self.layer1(x)).reshape(x.shape[0], -1))


@pytest.mark.gpu
def test_update_bn_on_the_convnet_matches_torch():
    torch.manual_seed(0)
    model = pdt.models.ConvNet().to(_dev())
    twin = _TorchConvNet().to(_dev())
    twin.load_state_dict(model.state_dict())
    g = torch.Generator(device=_dev()).manual_seed(4)
    loader = [torch.rand(100, 1, 28, 28, device=_dev(), generator=g) for _ in range(5)]
    psw.update_bn(loader, model)
    tsw.update_bn(loader, twin)
    for (n, a), b in zip(model.state_dict().items(), twin.state_dict().values()):
        if a.dtype == torch.int64:
            assert torch.equal(a, b) and a.item() == 5, n
        else:
            # the suite's TF32 tolerance (the convolutions run on TF32 tensor cores)
            assert (a - b).abs().max().item() <= 2e-2 * b.abs().max().item(), (n, (a - b).abs().max().item())
    assert model.layer1[1].momentum == 0.1   # update_bn restores the momentum


@pytest.mark.gpu
def test_checkpoint_round_trip_resumes_bit_identically(tmp_path):
    from pytorch_distributed_train_b200.utils import load_checkpoint, save_checkpoint

    def make():
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(_dev())
        opt = pdt.optim.SGD(model.parameters(), 0.05, momentum=0.9)
        return model, opt, psw.AveragedModel(model, multi_avg_fn=psw.get_ema_multi_avg_fn(0.8), use_buffers=True)

    g = torch.Generator(device=_dev()).manual_seed(2)
    batches = [(torch.rand(100, 1, 28, 28, device=_dev(), generator=g), torch.randint(0, 10, (100,), device=_dev(), generator=g))
               for _ in range(6)]

    def train(model, opt, avg, bs):
        for x, t in bs:
            opt.zero_grad()
            F.cross_entropy(model(x), t).backward()
            opt.step()
            avg.update_parameters(model)

    a = make()
    train(*a, batches)
    b = make()
    train(*b, batches[:3])
    ck = str(tmp_path / "ck.pt")
    save_checkpoint(ck, b[0], b[1], averaged_model=b[2])
    c = make()
    load_checkpoint(ck, c[0], c[1], averaged_model=c[2])
    assert c[2].n_averaged.item() == 3
    train(*c, batches[3:])
    _assert_same(c[2].state_dict(), a[2].state_dict())
    _assert_same(c[0].state_dict(), a[0].state_dict())


def _ddp_ema_n2(rank, world, port):
    import torch.distributed as td

    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    dev = torch.device("cuda", rank)
    g = torch.Generator().manual_seed(100 + rank)
    xs, ts = torch.rand(4, 100, 1, 28, 28, generator=g), torch.randint(0, 10, (4, 100), generator=g)
    torch.manual_seed(0)
    model = pdt.models.ConvNet().to(dev)
    avg = psw.AveragedModel(model, multi_avg_fn=psw.get_ema_multi_avg_fn(0.9), use_buffers=True)
    opt = pdt.optim.SGD(model.parameters(), 0.05)
    ddp = pdt.DistributedDataParallel(model, device_ids=[rank])
    step = GraphedTrainStep(ddp, pdt.nn.CrossEntropyLoss(), opt, (xs[0].to(dev), ts[0].to(dev)), warmup=3, averaged_model=avg)
    warm = 4   # GraphedTrainStep's warm-up steps with the fused SGD (max(warmup, 4))
    for i in range(8):
        step(xs[i % 4].pin_memory(), ts[i % 4].pin_memory())
    torch.cuda.synchronize()
    ours = torch.cat([p.detach().reshape(-1) for p in avg.module.parameters()]).cpu()

    td.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", world_size=world, rank=rank)
    try:
        torch.manual_seed(0)
        ref = pdt.models.ConvNet().to(dev)
        rddp = torch.nn.parallel.DistributedDataParallel(ref, device_ids=[rank])
        ropt = torch.optim.SGD(rddp.parameters(), 0.05)
        ravg = None
        for n, i in enumerate([0] * warm + [i % 4 for i in range(8)]):
            ropt.zero_grad()
            F.cross_entropy(rddp(xs[i].to(dev)), ts[i].to(dev)).backward()
            ropt.step()
            if n == warm:   # the first replay: GraphedTrainStep does not average its warm-up steps
                ravg = tsw.AveragedModel(ref, device=dev, multi_avg_fn=tsw.get_ema_multi_avg_fn(0.9), use_buffers=True)
            if ravg is not None:
                ravg.update_parameters(ref)
        theirs = torch.cat([p.detach().reshape(-1) for p in ravg.module.parameters()]).cpu()
    finally:
        td.destroy_process_group()
    return ours, theirs, step.kernels_per_replay


@pytest.mark.gpu
@pytest.mark.multigpu
def test_graphed_step_with_averaging_at_two_gpus_follows_torch_ddp():
    from mp_helpers import free_port, run_ranks

    res = run_ranks(_ddp_ema_n2, 2, free_port(), backend="nccl")
    assert torch.equal(res[0][0], res[1][0]), "ranks must stay bit-identical"
    for ours, theirs, _ in res:
        err = (ours - theirs).abs().max().item() / theirs.abs().max().item()
        assert err < 2e-2, err
