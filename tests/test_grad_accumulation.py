"""Gradient accumulation: GraphedTrainStep(accumulation_steps=k) — k micro-batches accumulated inside the two fused backward kernels
with the update riding on the last one — against float64, against pdt's own eager loop bit for bit, against torch's optimizers,
its fallback configurations through autograd, and train_mnist.py --accumulation-steps against torch DDP with no_sync."""
import contextlib
import copy
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import pytorch_distributed_train_b200 as pdt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# =====================================================================================================================
# CPU
# =====================================================================================================================
def test_cli_validates_accumulation_steps():
    from pytorch_distributed_train_b200 import cli

    assert cli.build_parser().parse_args([]).accumulation_steps == 1
    for argv, msg in ((["--accumulation-steps", "0"], "--accumulation-steps must be at least 1"),
                      (["--accumulation-steps", "-2"], "--accumulation-steps must be at least 1"),
                      (["--graph", "-g", "2", "--accumulation-steps", "2"], "runs on one GPU only")):
        out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py")] + argv, capture_output=True, text=True, timeout=60,
                             cwd=ROOT)
        assert out.returncode != 0 and msg in out.stderr, (argv, out.stderr[-500:])
    p = cli.build_parser()
    cli.check_args(p, p.parse_args(["--graph", "--accumulation-steps", "4"]))   # one GPU: accepted
    cli.check_args(p, p.parse_args(["-g", "2", "--accumulation-steps", "4"]))   # eager loop: accepted


def _torch_ddp_accum(rank, world, port, steps, lr, k, max_norm, div):
    """torch DDP + gloo on train_mnist.py's data, model and seed: k micro-batches of 100 per step, no_sync on all but the last,
    each backward of loss / div (div = k: torch's convention), then — with max_norm — torch.nn.utils.clip_grad_norm_ of the
    accumulated gradients.  Returns the final state and the pre-clip norm of every step."""
    import torch.distributed as td

    from pytorch_distributed_train_b200 import data as pdata

    td.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", world_size=world, rank=rank)
    try:
        torch.manual_seed(0)
        model = pdt.models.ConvNet()
        ddp = torch.nn.parallel.DistributedDataParallel(model)
        opt = torch.optim.SGD(ddp.parameters(), lr)
        crit = torch.nn.CrossEntropyLoss()
        ds = pdata.SyntheticMNIST(1200, seed=0, num_classes=10, image_shape=(1, 28, 28))
        loader = torch.utils.data.DataLoader(ds, batch_size=100 * k, shuffle=False,
                                             sampler=torch.utils.data.DistributedSampler(ds, num_replicas=world, rank=rank))
        norms = []
        for i, (x, y) in enumerate(loader):
            if i >= steps:
                break
            opt.zero_grad()
            for j, (xm, ym) in enumerate(zip(x.split(100), y.split(100))):
                with ddp.no_sync() if j + 1 < k else contextlib.nullcontext():
                    (crit(ddp(xm), ym) / div).backward()
            if max_norm is not None:
                norms.append(torch.nn.utils.clip_grad_norm_(ddp.parameters(), max_norm).item())
            opt.step()
        return {n: v.clone() for n, v in ddp.state_dict().items()}, norms
    finally:
        td.destroy_process_group()


def _close(ours, ref):
    return all(torch.allclose(ours[n].float(), ref[n].float(), atol=1e-5, rtol=1e-4) for n in ref)


# lr 0.1 without clipping is dominated by float32 summation-order noise (it exceeds the tolerance without accumulation too); lr 0.02
# keeps that noise well inside it while a wrong 1/K moves the weights far outside
@pytest.mark.parametrize("lr,clip", [(0.02, None), (0.1, 0.5)])
def test_train_script_accumulation_matches_torch_ddp_gloo(tmp_path, lr, clip):
    from mp_helpers import free_port, run_ranks

    ck = str(tmp_path / "accum.pt")
    cmd = [sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "2", "--backend", "gloo", "--lr", str(lr), "--accumulation-steps", "2",
           "--steps", "3", "--samples", "1200", "--epochs", "1", "--log-interval", "3", "--checkpoint", ck]
    if clip is not None:
        cmd += ["--clip-grad-norm", str(clip)]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=240, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "Epoch [1/1], Step [3/3]" in out.stdout   # optimizer steps: 600 images per rank in loader batches of 2 × 100
    ours = torch.load(ck, map_location="cpu", weights_only=False)["model"]
    ref, norms = run_ranks(_torch_ddp_accum, 2, free_port(), 3, lr, 2, clip, 2)[0]
    assert list(ours) == list(ref)
    for n in ref:
        assert torch.allclose(ours[n].float(), ref[n].float(), atol=1e-5, rtol=1e-4), (n, (ours[n].float() - ref[n].float()).abs().max())
    if clip is None:
        # the comparison sees the scale: a loop without the / 2 ends outside the tolerance
        wrong, _ = run_ranks(_torch_ddp_accum, 2, free_port(), 3, lr, 2, None, 1)[0]
        assert not _close(ours, wrong)
    else:
        assert min(norms) > clip, norms   # clipping engaged on every step


# =====================================================================================================================
# GPU
# =====================================================================================================================
def _dev():
    return torch.device("cuda", 0)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@contextlib.contextmanager
def _one_gpu():
    from mp_helpers import free_port

    torch.cuda.set_device(0)
    pdt.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{free_port()}", world_size=1, rank=0)
    try:
        yield
    finally:
        pdt.destroy_process_group()


def _batch(k, b, seed):
    g = torch.Generator(device=_dev()).manual_seed(seed)
    return torch.rand(k * b, 1, 28, 28, device=_dev(), generator=g), torch.randint(0, 10, (k * b,), device=_dev(), generator=g)


def _float64_accumulated(model, x, t, k):
    """A float64 torch twin of `model`'s current state fed the same k micro-batches, each backward of loss / k."""
    ref = pdt.models.ConvNet(fused=False).to(_dev())
    ref.load_state_dict(model.state_dict())
    ref = ref.double()
    b = x.shape[0] // k
    for i in range(k):
        (F.cross_entropy(ref(x[i * b:(i + 1) * b].double()), t[i * b:(i + 1) * b]) / k).backward()
    return ref


def _rel(ours, ref):
    """bench.py's verification metric: max |ours − reference| / max |reference| over the flat vector."""
    ours = torch.cat([o.double().reshape(-1) for o in ours])
    ref = torch.cat([r.double().reshape(-1) for r in ref])
    return (ours - ref).abs().max().item() / ref.abs().max().item()


def _assert_grads_match_float64(model, ref):
    # a frozen parameter gets no gradient (the twin computes every one)
    assert all(p.grad is None for p in model.parameters() if not p.requires_grad)
    refs = dict(ref.named_parameters())
    named = [(n, p, refs[n]) for n, p in model.named_parameters() if p.requires_grad]
    # conv biases feed a BatchNorm: their true gradient is zero and what is left is rounding noise
    keep = [(p, q) for n, p, q in named if n not in ("layer1.0.bias", "layer2.0.bias")]
    err = _rel([p.grad for p, _ in keep], [q.grad for _, q in keep])
    assert err < 2e-2, err
    for n, p, q in named:
        if n in ("layer1.0.bias", "layer2.0.bias"):
            assert (p.grad.double() - q.grad).abs().max().item() < 1e-4, n


def _assert_loss_is_mean(loss, state, x, t, k):
    """The step's loss is the mean of the k micro-batch losses of the model in `state`, in float64."""
    b = x.shape[0] // k
    with torch.no_grad():
        twin = pdt.models.ConvNet(fused=False).to(_dev())
        twin.load_state_dict(state)
        twin = twin.double()
        losses = [F.cross_entropy(twin(x[i * b:(i + 1) * b].double()), t[i * b:(i + 1) * b]).item() for i in range(k)]
    assert abs(loss.item() - sum(losses) / k) < 2e-3, (loss.item(), losses)


def _graphed(model, opt, x, t, k, **kw):
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    ddp = pdt.DistributedDataParallel(model, device_ids=[0])
    return GraphedTrainStep(ddp, pdt.nn.CrossEntropyLoss(), opt, (x, t), warmup=2, accumulation_steps=k, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [2, 3, 4])
@pytest.mark.parametrize("b", ["100", "sms"])
def test_accumulated_gradients_match_float64(k, b):
    b = _sms() if b == "sms" else int(b)
    with _one_gpu():
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(_dev())
        opt = pdt.optim.SGD(model.parameters(), lr=0.0)
        x, t = _batch(k, b, 5)
        step = _graphed(model, opt, x, t, k)
        assert step.accumulates_in_kernel and step.kernels_per_replay == 3 * k, step.kernels_per_replay
        x, t = _batch(k, b, 6)
        before = {n: v.clone() for n, v in model.state_dict().items()}
        ref = _float64_accumulated(model, x, t, k)   # its BatchNorm buffers advance k times as well
        loss = step(x, t)
        torch.cuda.synchronize()
        _assert_grads_match_float64(model, ref)
        _assert_loss_is_mean(loss, before, x, t, k)   # static_loss: the mean of the k micro-batch losses
        for (n, v), (_, r) in zip(model.named_buffers(), ref.named_buffers()):
            if n.endswith("num_batches_tracked"):
                assert int(v) == int(r) == int(before[n]) + k, n
            else:
                assert torch.allclose(v.double(), r, atol=2e-3, rtol=1e-3), (n, (v.double() - r).abs().max().item())
        for n, p in model.named_parameters():
            assert torch.equal(p.detach(), before[n]), n   # lr = 0


@pytest.mark.gpu
@pytest.mark.parametrize("k", [2, 4])
def test_accumulated_gradients_equal_eager_loop_bitwise(k):
    """1/k is exact for k = 2, 4: the in-kernel accumulation equals pdt's eager loop, in which autograd adds the temporaries."""
    from pytorch_distributed_train_b200.ops import functional as OF

    with _one_gpu():
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(_dev())
        opt = pdt.optim.SGD(model.parameters(), lr=0.0)
        x, t = _batch(k, 100, 7)
        step = _graphed(model, opt, x, t, k)
        assert step.accumulates_in_kernel
        x, t = _batch(k, 100, 8)
        eager = pdt.models.ConvNet().to(_dev())
        eager.load_state_dict(model.state_dict())
        step(x, t)
        crit = pdt.nn.CrossEntropyLoss()
        for i in range(k):
            xi, ti = x[i * 100:(i + 1) * 100], t[i * 100:(i + 1) * 100]
            with OF.upcoming_targets(ti):
                out = eager(xi)
            (crit(out, ti) / k).backward()
        torch.cuda.synchronize()
        for (n, p), q in zip(model.named_parameters(), eager.parameters()):
            assert torch.equal(p.grad, q.grad), (n, (p.grad - q.grad).abs().max().item())


@pytest.mark.gpu
@pytest.mark.parametrize("optim", ["sgd", "adamw"])
@pytest.mark.parametrize("clip", [None, 0.5])
def test_graphed_accumulation_follows_torch(optim, clip):
    k, b = 2, 100
    with _one_gpu():
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(_dev())
        if optim == "sgd":
            opt = pdt.optim.SGD(model.parameters(), 0.05, momentum=0.9)
        else:
            opt = pdt.optim.AdamW(model.parameters(), 1e-3)
        xs = [_batch(k, b, 20 + i) for i in range(4)]
        step = _graphed(model, opt, xs[0][0], xs[0][1], k, max_grad_norm=clip)
        assert step.accumulates_in_kernel and step.kernels_per_replay == 3 * k, step.kernels_per_replay
        # the reference starts where the engine's eager warm-up steps left the model and the optimizer
        ref = pdt.models.ConvNet().to(_dev())
        ref.load_state_dict(model.state_dict())
        if optim == "sgd":
            ropt = torch.optim.SGD(ref.parameters(), 0.05, momentum=0.9, foreach=False)
        else:
            ropt = torch.optim.AdamW(ref.parameters(), 1e-3, foreach=False)
        ropt.load_state_dict(copy.deepcopy(opt.state_dict()))   # torch would otherwise share our state tensors
        steps0 = [float(st["step"]) for st in opt.state.values()] if optim == "adamw" else None
        crit = pdt.nn.CrossEntropyLoss()
        for r in range(10):
            x, t = xs[r % 4]
            step(x, t)
            ropt.zero_grad()
            for i in range(k):
                (crit(ref(x[i * b:(i + 1) * b]), t[i * b:(i + 1) * b]) / k).backward()
            norm = torch.nn.utils.clip_grad_norm_(ref.parameters(), clip) if clip is not None else None
            if r == 0 and clip is not None:
                torch.cuda.synchronize()
                # the norm of the accumulated gradients, from the same state
                assert abs(step.grad_norm.item() - norm.item()) <= 1e-3 * norm.item(), (step.grad_norm.item(), norm.item())
            ropt.step()
        torch.cuda.synchronize()
        if optim == "adamw":
            assert all(float(st["step"]) == s + 10 for st, s in zip(opt.state.values(), steps0))   # once per replay
        keep = [(p, q) for (n, p), q in zip(model.named_parameters(), ref.parameters()) if n not in ("layer1.0.bias", "layer2.0.bias")]
        err = _rel([p.detach() for p, _ in keep], [q.detach() for _, q in keep])
        assert err < 2e-2, err


@pytest.mark.gpu
def test_replay_has_no_add_and_no_optimizer_kernel():
    from torch.profiler import ProfilerActivity, profile

    k = 2
    with _one_gpu():
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(_dev())
        opt = pdt.optim.SGD(model.parameters(), 0.01, momentum=0.9)
        x, t = _batch(k, 100, 30)
        step = _graphed(model, opt, x, t, k, max_grad_norm=1.0)
        step(x, t)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step(x, t)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        kernels = [n for n in names if "memcpy" not in n.lower() and "memset" not in n.lower()]
        assert not [n for n in kernels if "elementwise" in n or "add" in n.lower().replace("grad", "")], kernels
        assert not [n for n in kernels if any(s in n for s in ("sgd_multi", "adam_multi", "grad_norm", "grad_scale"))], kernels
        assert sum("convnet_" in n for n in kernels) == 3 * k, kernels


def _times_one(crit):
    return lambda o, t: crit(o, t) * 1.0


def _plus_zero_reg(crit):
    return lambda o, t: crit(o, t) + 0.0 * o.square().mean()


@pytest.mark.gpu
@pytest.mark.parametrize("wrap", [_times_one, _plus_zero_reg])
def test_criterion_wrapping_the_cross_entropy_is_scaled_once(wrap):
    """A criterion that computes something from pdt's cross-entropy must see the unscaled value: the forward kernel does not
    pre-scale it, each micro-batch backpropagates loss / k through autograd, and the gradients and the step's loss match float64."""
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    k, b = 2, 100
    with _one_gpu():
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(_dev())
        opt = pdt.optim.SGD(model.parameters(), lr=0.0)
        x, t = _batch(k, b, 70)
        ddp = pdt.DistributedDataParallel(model, device_ids=[0])
        step = GraphedTrainStep(ddp, wrap(pdt.nn.CrossEntropyLoss()), opt, (x, t), warmup=2, accumulation_steps=k)
        assert not step.accumulates_in_kernel
        x, t = _batch(k, b, 71)
        before = {n: v.clone() for n, v in model.state_dict().items()}
        ref = _float64_accumulated(model, x, t, k)
        loss = step(x, t)
        torch.cuda.synchronize()
        _assert_grads_match_float64(model, ref)
        _assert_loss_is_mean(loss, before, x, t, k)


@pytest.mark.gpu
def test_criterion_that_stops_returning_the_cross_entropy_is_refused():
    """The kernel's 1/k is armed by a first step whose criterion returned the cross-entropy unchanged; a criterion that wraps it later
    would get the scale twice and is refused."""
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    crit = pdt.nn.CrossEntropyLoss()
    calls = []

    def fickle(o, t):
        calls.append(1)
        return crit(o, t) if len(calls) <= 2 else crit(o, t) * 1.0

    with _one_gpu():
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(_dev())
        opt = pdt.optim.SGD(model.parameters(), lr=0.0)
        x, t = _batch(2, 100, 72)
        ddp = pdt.DistributedDataParallel(model, device_ids=[0])
        with pytest.raises(RuntimeError, match="scale would be applied twice"):
            GraphedTrainStep(ddp, fickle, opt, (x, t), warmup=2, accumulation_steps=2)


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["PDT_FUSED_LAYERS", "above_sms", "frozen_conv1"])
def test_fallback_configurations_accumulate_through_autograd(config, monkeypatch):
    k = 2
    b = _sms() + 18 if config == "above_sms" else 100
    if config == "PDT_FUSED_LAYERS":
        monkeypatch.setenv(config, "0")
    with _one_gpu():
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(_dev())
        if config == "frozen_conv1":   # a partially trainable model takes the per-op kernels
            model.layer1[0].requires_grad_(False)
        opt = pdt.optim.SGD(model.parameters(), lr=0.0)
        x, t = _batch(k, b, 40)
        step = _graphed(model, opt, x, t, k)
        assert not step.accumulates_in_kernel
        x, t = _batch(k, b, 41)
        before = {n: v.clone() for n, v in model.state_dict().items()}
        ref = _float64_accumulated(model, x, t, k)
        loss = step(x, t)
        torch.cuda.synchronize()
        _assert_grads_match_float64(model, ref)
        _assert_loss_is_mean(loss, before, x, t, k)


_K1_ARM = """
import sys, torch
sys.path.insert(0, {tests!r})
import pytorch_distributed_train_b200 as pdt
from pytorch_distributed_train_b200.engine import GraphedTrainStep
from mp_helpers import free_port

torch.cuda.set_device(0)
pdt.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{{free_port()}}", world_size=1, rank=0)
dev = torch.device("cuda", 0)
def batch(seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.rand(100, 1, 28, 28, device=dev, generator=g), torch.randint(0, 10, (100,), device=dev, generator=g)
torch.manual_seed(0)
model = pdt.models.ConvNet().to(dev)
opt = pdt.optim.SGD(model.parameters(), 0.05, momentum=0.9)
ddp = pdt.DistributedDataParallel(model, device_ids=[0])
step = GraphedTrainStep(ddp, pdt.nn.CrossEntropyLoss(), opt, batch(50), warmup=2, **{kw})
assert step.kernels_per_replay == 3
for r in range(3):
    step(*batch(51 + r))
torch.cuda.synchronize()
torch.save([p.detach().cpu() for p in model.parameters()], {out!r})
pdt.destroy_process_group()
"""


@pytest.mark.gpu
def test_one_accumulation_step_is_the_plain_step(tmp_path):
    """accumulation_steps=1 is today's step: the parameters after three replays equal, bit for bit, those of a step constructed without
    the argument.  Each arm runs in a fresh process, so that both start from the same process state."""
    params = []
    for i, kw in enumerate(({}, {"accumulation_steps": 1})):
        out = str(tmp_path / f"arm{i}.pt")
        code = _K1_ARM.format(tests=os.path.join(ROOT, "tests"), kw=kw, out=out)
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=240, cwd=ROOT)
        assert r.returncode == 0, r.stderr[-2000:]
        params.append(torch.load(out))
    names = [n for n, _ in pdt.models.ConvNet().named_parameters()]
    for n, p, q in zip(names, *params):
        assert torch.equal(p, q), n


@pytest.mark.gpu
def test_engine_rejects_bad_accumulation_arguments():
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    model = pdt.models.ConvNet().to(_dev())
    opt = pdt.optim.SGD(model.parameters(), 0.01)
    x, t = _batch(1, 100, 60)
    for k in (0, -1, 1.5, 3):   # 100 rows do not split into 3 micro-batches
        with pytest.raises(ValueError):
            GraphedTrainStep(model, pdt.nn.CrossEntropyLoss(), opt, (x, t), accumulation_steps=k)
