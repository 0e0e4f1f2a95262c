"""Class-probability targets on the native cross-entropy: the stand-alone kernels, the forward kernel's loss rider, the routing of
what they do not take to torch, the graphed training step (with in-kernel accumulation) and train_mnist.py --mixup on the GPU.
The oracle is F.cross_entropy in float64 on the CPU, with test_cross_entropy_options.py's tolerances."""
import contextlib
import copy
import math
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import pytorch_distributed_train_b200 as pdt
from pytorch_distributed_train_b200 import _C
from pytorch_distributed_train_b200.ops import functional as OF

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_torch_ce = F.cross_entropy   # the oracle, kept before a test makes the native path's fall-back raise


@pytest.fixture
def no_torch_ce(monkeypatch):
    """Every cross-entropy under test must run on the native kernels: torch's functional raises if it is reached."""
    def _raise(*a, **k):
        raise AssertionError("F.cross_entropy was called")

    monkeypatch.setattr(torch.nn.functional, "cross_entropy", _raise)


def dev():
    return torch.device("cuda", 0)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _weights(kind, C, gen):
    if kind == "none":
        return None
    w = torch.rand(C, generator=gen) + 0.25
    if kind == "some_zero":
        w[::3] = 0.0
    return w.to(dev())


def _probs(kind, B, C, gen):
    """fp32 [B, C] targets of one kind, on the device."""
    y = torch.randint(0, C, (B,), generator=gen)
    onehot = F.one_hot(y, C).float()
    if kind == "onehot":
        q = onehot
    elif kind == "dirichlet":   # Dirichlet(1, …, 1): normalised exponentials
        e = -torch.log(torch.rand(B, C, generator=gen).clamp_min(1e-12))
        q = e / e.sum(1, keepdim=True)
    elif kind == "twohot":      # MixUp: λ·onehot(y) + (1 − λ)·onehot of the previous row
        lam = torch.rand(B, 1, generator=gen)
        q = lam * onehot + (1 - lam) * onehot.roll(1, 0)
    elif kind == "unnormalised":
        q = 2 * torch.randn(B, C, generator=gen)
    else:
        assert kind == "zeros"
        q = torch.zeros(B, C)
    return q.contiguous().to(dev())


KINDS = ("onehot", "dirichlet", "twohot", "unnormalised", "zeros")


def _reference(x, q, w, reduction, eps, scale=1.0):
    """Loss and scale · d(loss)/d(logits) in float64 on the CPU, and the magnitudes the fp32 sums carry: Σ_c |a_c|·|lse − x_c| / D
    for the loss and (p_c·Σ_k |a_k| + |a_c|)·scale / D for the gradient, a_c = w_c·q'_c."""
    xd = x.detach().double().cpu().requires_grad_()
    qd = q.double().cpu()
    wd = None if w is None else w.double().cpu()
    loss = _torch_ce(xd, qd, wd, reduction=reduction, label_smoothing=eps)
    (g,) = torch.autograd.grad(loss * scale, xd)
    C = x.shape[1]
    a = (qd * (1 - eps) + eps / C) * (1.0 if wd is None else wd)
    D = 1.0 if reduction == "sum" else float(x.shape[0])
    lsm = torch.log_softmax(xd.detach(), 1)
    loss_mag = float((a.abs() * lsm.abs()).sum()) / D if D else 0.0
    grad_mag = (lsm.exp() * a.abs().sum(1, keepdim=True) + a.abs()) * abs(scale) / D if D else torch.zeros_like(g)
    return loss.detach(), g, loss_mag, grad_mag


def _assert_loss(got, ref, mag):
    if math.isnan(ref.item()):
        assert math.isnan(got.item()), got.item()
    else:
        assert abs(got.item() - ref.item()) <= 1e-5 * max(abs(ref.item()), mag) + 1e-6, (got.item(), ref.item(), mag)


def _assert_grad(got, ref, mag):
    got = got.double().cpu()
    size = max(ref.abs().max().item(), mag.max().item()) if ref.numel() else 0.0
    if size == 0.0:
        assert torch.equal(got, torch.zeros_like(got))
        return
    assert torch.allclose(got, ref, rtol=1e-5, atol=1e-6 * size), (got - ref).abs().max().item()


# ---- 1. stand-alone kernels -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("eps", [0.0, 0.1, 1.0])
@pytest.mark.parametrize("C", [1, 2, 10, 1024])
@pytest.mark.parametrize("B", [1, 7, 100, 300])
def test_standalone_kernels_match_float64(B, C, eps, no_torch_ce):
    gen = torch.Generator().manual_seed(B * 7 + C)
    x = torch.randn(B, C, generator=gen).to(dev())
    for wkind in ("none", "random", "some_zero"):
        w = _weights(wkind, C, gen)
        for reduction in ("mean", "sum"):
            crit = pdt.nn.CrossEntropyLoss(weight=w, reduction=reduction, label_smoothing=eps)
            for kind in KINDS:
                q = _probs(kind, B, C, gen)
                case = (wkind, reduction, kind)
                for scale in (1.0, 3.0):
                    ref_loss, ref_g, loss_mag, grad_mag = _reference(x, q, w, reduction, eps, scale)
                    xs = x.clone().requires_grad_()
                    loss = crit(xs, q)
                    (loss if scale == 1.0 else loss * scale).backward()
                    try:
                        _assert_loss(loss, ref_loss, loss_mag)
                        _assert_grad(xs.grad, ref_g, grad_mag)
                    except AssertionError as e:
                        raise AssertionError(f"{case} scale {scale}: {e}") from None
                # the saved gradient for a unit incoming gradient, and the separate backward kernel from the saved softmax with an
                # incoming gradient of 3
                ref_loss, ref_g1, loss_mag, grad_mag1 = _reference(x, q, w, reduction, eps)
                loss, g1 = _C.cross_entropy_fwd(x, q, True, w, -100, eps, reduction)
                _assert_loss(loss, ref_loss, loss_mag)
                _assert_grad(g1, ref_g1, grad_mag1)
                loss, probs = _C.cross_entropy_fwd(x, q, False, w, -100, eps, reduction)
                _assert_loss(loss, ref_loss, loss_mag)
                assert torch.allclose(probs.double(), torch.softmax(x.double(), 1), rtol=1e-5, atol=1e-7), case
                g = _C.cross_entropy_bwd(probs, q, torch.tensor(3.0, device=dev()), w, -100, eps, reduction)
                _assert_grad(g, ref_g, grad_mag)


def test_standalone_kernels_are_reproducible_and_empty_mean_is_nan():
    gen = torch.Generator().manual_seed(1)
    x = torch.randn(300, 1024, generator=gen).to(dev())
    q = _probs("dirichlet", 300, 1024, gen)
    a = _C.cross_entropy_fwd(x, q, True, None, -100, 0.1, "mean")
    b = _C.cross_entropy_fwd(x, q, True, None, -100, 0.1, "mean")
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    e = torch.empty(0, 10, device=dev())
    loss, _ = _C.cross_entropy_fwd(e, e, True, None, -100, 0.0, "mean")
    assert math.isnan(loss.item()) and math.isnan(_torch_ce(e.cpu(), e.cpu()).item())
    loss, _ = _C.cross_entropy_fwd(e, e, True, None, -100, 0.0, "sum")
    assert loss.item() == 0.0
    assert _C.cross_entropy_bwd(e, e, torch.tensor(1.0, device=dev())).shape == (0, 10)


def test_bindings_reject_bad_probability_targets():
    x = torch.randn(4, 10, device=dev())
    q = torch.softmax(torch.randn(4, 10, device=dev()), 1)
    with pytest.raises(RuntimeError, match="ignore_index"):
        _C.cross_entropy_fwd(x, q, True, None, 3, 0.0, "mean")
    with pytest.raises(RuntimeError, match="ignore_index"):
        _C.cross_entropy_bwd(x, q, torch.tensor(1.0, device=dev()), None, 3, 0.0, "mean")
    with pytest.raises(RuntimeError, match="shape"):
        _C.cross_entropy_fwd(x, q[:, :9].contiguous(), True)
    with pytest.raises(RuntimeError, match="dtype"):
        _C.cross_entropy_fwd(x, q.double(), True)
    with pytest.raises(RuntimeError, match="contiguous"):
        _C.cross_entropy_fwd(x, q.t().contiguous().t(), True)
    with pytest.raises(RuntimeError, match="CUDA"):
        _C.cross_entropy_fwd(x, q.cpu(), True)


# ---- 2. the forward kernel's loss rider -------------------------------------------------------------------------------------------
_SPECS = {
    "plain": dict(),
    "smooth_weighted": dict(label_smoothing=0.1, weight="random"),
    "sum_zero_weights": dict(reduction="sum", weight="some_zero"),
}


@pytest.mark.parametrize("late", [False, True])
@pytest.mark.parametrize("scale", [1.0, 0.25])
@pytest.mark.parametrize("B", ["1", "2", "100", "sms"])
@pytest.mark.parametrize("ncls", [1, 2, 10, 16])
def test_forward_kernel_rider_matches_float64_and_standalone_kernel(ncls, B, scale, late):
    B = sms() if B == "sms" else int(B)
    torch.manual_seed(3)
    net = pdt.models.ConvNet(num_classes=ncls, fused=True).to(dev())
    gen = torch.Generator().manual_seed(ncls * 1000 + B)
    x = torch.rand(B, 1, 28, 28, generator=gen).to(dev())
    for name, kw in _SPECS.items():
        kw = dict(kw)
        if "weight" in kw:
            kw["weight"] = _weights(kw["weight"], ncls, gen)
        crit = pdt.nn.CrossEntropyLoss(**kw)
        for kind in ("twohot", "unnormalised"):
            q = _probs(kind, B, ncls, gen)
            with OF.upcoming_targets(q, loss_read_after_backward=late, grad_scale=scale, spec=OF.ce_spec_of(crit)):
                out = net(x)
            pre = getattr(out, "_pdt_ce", None)
            assert pre is not None and pre[0] is q, (name, kind)
            loss = crit(out, q)
            assert getattr(loss, "_pdt_loss_scale", None) == scale   # the rider's loss, not the stand-alone kernel's
            loss.backward()
            dlogits = pre[2]
            ref_loss, ref_g, loss_mag, grad_mag = _reference(out, q, crit.weight, crit.reduction, crit.label_smoothing, scale)
            case = (name, kind)
            try:
                _assert_loss(loss / scale, ref_loss, loss_mag)
                _assert_grad(dlogits, ref_g, grad_mag)
                # the stand-alone kernel on the same logits: the same formula summed in another order
                sl, sg = _C.cross_entropy_fwd(out.detach(), q, True, crit.weight, -100, crit.label_smoothing, crit.reduction)
                assert abs(loss.item() / scale - sl.item()) <= 1e-5 * max(abs(sl.item()), loss_mag) + 1e-6, (loss.item(), sl.item())
                _assert_grad(dlogits / scale, sg.double().cpu(), grad_mag / scale)
            except AssertionError as e:
                raise AssertionError(f"{case}: {e}") from None
            net.zero_grad(set_to_none=True)


# ---- 3. what the native paths do not take goes to torch ---------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["fp64", "fp16", "non_contiguous", "wrong_shape", "ignore_index", "none_reduction", "unbatched"])
def test_other_probability_targets_reach_torch(case, monkeypatch):
    calls = []

    def _counting(*a, **k):
        calls.append(1)
        return _torch_ce(*a, **k)

    monkeypatch.setattr(torch.nn.functional, "cross_entropy", _counting)
    gen = torch.Generator().manual_seed(2)
    x = torch.randn(6, 10, generator=gen).to(dev())
    q = torch.softmax(torch.randn(6, 10, generator=gen), 1).to(dev())
    kw = dict(label_smoothing=0.1)
    if case == "fp64":
        q = q.double()
    elif case == "fp16":
        q = q.half()
    elif case == "non_contiguous":
        q = torch.softmax(torch.randn(10, 6, generator=gen), 0).to(dev()).t()
        assert not q.is_contiguous()
    elif case == "wrong_shape":
        q = q[:, :9]
    elif case == "ignore_index":
        kw["ignore_index"] = 3
    elif case == "unbatched":   # a [C] input with a [C] target
        x, q = x[0], q[0]
    else:
        kw["reduction"] = "none"
    crit = pdt.nn.CrossEntropyLoss(**kw)
    assert not crit.native_ok(x, q)
    try:
        want = _torch_ce(x, q, **kw)
    except Exception as e:   # torch's error, raised again through pdt's criterion
        with pytest.raises(type(e)):
            crit(x, q)
        assert calls
        return
    got = crit(x, q)
    assert calls and torch.allclose(got, want), (got, want)


def test_rider_stays_off_for_ignore_index():
    """The forward kernel takes probability targets only with the default ignore_index (torch refuses the others)."""
    torch.manual_seed(3)
    net = pdt.models.ConvNet(fused=True).to(dev())
    x = torch.rand(8, 1, 28, 28, device=dev())
    q = torch.softmax(torch.randn(8, 10, device=dev()), 1)
    with OF.upcoming_targets(q, spec=(None, 3, "mean", 0.0)):
        out = net(x)
    assert getattr(out, "_pdt_ce", None) is None
    with OF.upcoming_targets(q, spec=(None, -100, "mean", 0.0)):
        out = net(x)
    assert out._pdt_ce[0] is q


# ---- 4. the graphed training step -------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _one_gpu():
    from mp_helpers import free_port

    torch.cuda.set_device(0)
    pdt.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{free_port()}", world_size=1, rank=0)
    try:
        yield
    finally:
        pdt.destroy_process_group()


def _batch(n, seed):
    """Images and MixUp-like targets (two non-zeros per row)."""
    gen = torch.Generator().manual_seed(seed)
    return torch.rand(n, 1, 28, 28, generator=gen).to(dev()), _probs("twohot", n, 10, gen)


def _rel(ours, ref):
    ours = torch.cat([o.double().reshape(-1) for o in ours])
    ref = torch.cat([r.double().reshape(-1) for r in ref])
    return (ours - ref).abs().max().item() / ref.abs().max().item()


def _smoothed_weighted():
    w = torch.rand(10, generator=torch.Generator().manual_seed(9)).to(dev()) + 0.25
    return pdt.nn.CrossEntropyLoss(label_smoothing=0.1, weight=w)


@pytest.mark.parametrize("optim", ["sgd", "adamw_clip"])
def test_graphed_step_with_soft_targets_follows_eager_loop(optim, no_torch_ce):
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    with _one_gpu():
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(dev())
        crit = _smoothed_weighted()
        clip = 0.5 if optim == "adamw_clip" else None
        opt = pdt.optim.SGD(model.parameters(), 0.05, momentum=0.9) if optim == "sgd" else pdt.optim.AdamW(model.parameters(), 1e-3)
        xs = [_batch(100, 40 + i) for i in range(4)]
        step = GraphedTrainStep(pdt.DistributedDataParallel(model, device_ids=[0]), crit, opt, xs[0], warmup=2, max_grad_norm=clip)
        assert step.kernels_per_replay == 3, step.kernels_per_replay
        # the eager loop starts where the engine's warm-up steps left the model and the optimizer; its loss is what
        # torch.nn.CrossEntropyLoss(weight, label_smoothing=0.1) computes (torch's functional, which the fixture hides from pdt)
        ref = pdt.models.ConvNet().to(dev())
        ref.load_state_dict(model.state_dict())
        if optim == "sgd":
            ropt = torch.optim.SGD(ref.parameters(), 0.05, momentum=0.9, foreach=False)
        else:
            ropt = torch.optim.AdamW(ref.parameters(), 1e-3, foreach=False)
        ropt.load_state_dict(copy.deepcopy(opt.state_dict()))   # torch would otherwise share our state tensors
        for r in range(8):
            x, q = xs[r % 4]
            loss = step(x, q)
            ropt.zero_grad()
            lr_ = _torch_ce(ref(x), q, crit.weight, label_smoothing=0.1)
            lr_.backward()
            if clip is not None:
                torch.nn.utils.clip_grad_norm_(ref.parameters(), clip)
            ropt.step()
            if r == 0:
                torch.cuda.synchronize()
                assert abs(loss.item() - lr_.item()) <= 1e-4 * abs(lr_.item()), (loss.item(), lr_.item())
        torch.cuda.synchronize()
        keep = [(p, q) for (n, p), q in zip(model.named_parameters(), ref.parameters()) if n not in ("layer1.0.bias", "layer2.0.bias")]
        err = _rel([p.detach() for p, _ in keep], [q.detach() for _, q in keep])
        assert err < 2e-2, err


@pytest.mark.parametrize("k", [2, 4])
def test_graphed_accumulation_with_soft_targets_accumulates_in_kernel(k, no_torch_ce):
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    class ThroughAutograd(GraphedTrainStep):
        _accumulate_in_kernel = False

    with _one_gpu():
        crit = _smoothed_weighted()
        torch.manual_seed(0)
        models = [pdt.models.ConvNet().to(dev()) for _ in range(2)]
        models[1].load_state_dict(models[0].state_dict())
        xs = [_batch(k * 100, 50 + i) for i in range(3)]
        steps = []
        for cls, m in zip((GraphedTrainStep, ThroughAutograd), models):
            opt = pdt.optim.SGD(m.parameters(), 0.05)
            steps.append(cls(pdt.DistributedDataParallel(m, device_ids=[0]), crit, opt, xs[0], warmup=2, accumulation_steps=k))
        assert steps[0].accumulates_in_kernel and steps[0].kernels_per_replay == 3 * k, steps[0].kernels_per_replay
        assert not steps[1].accumulates_in_kernel
        for r in range(4):
            la, lb = (s(*xs[r % 3]) for s in steps)
            torch.cuda.synchronize()
            assert abs(la.item() - lb.item()) <= 1e-6 * abs(lb.item()), (r, la.item(), lb.item())
        for (n, p), q in zip(models[0].named_parameters(), models[1].parameters()):
            assert torch.allclose(p, q, rtol=1e-5, atol=1e-6), (n, (p - q).abs().max().item())


# ---- 5. train_mnist.py --mixup on the GPU -----------------------------------------------------------------------------------------
def test_train_script_with_mixup_in_graphed_step():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "1", "--graph", "--mixup", "0.2", "--steps", "20",
                          "--samples", "4000", "--epochs", "1", "--log-interval", "5"],
                         capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    losses = [float(v) for v in re.findall(r"Step \[\d+/\d+\], Loss: (\S+)", out.stdout)]
    assert len(losses) == 4 and all(math.isfinite(v) for v in losses), out.stdout[-1000:]
