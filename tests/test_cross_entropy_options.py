"""torch's cross-entropy options on the native kernels: class weights, label smoothing, any ignore_index and the sum reduction, in the
stand-alone kernels, in the forward kernel's loss rider, and in the graphed training step.  The oracle is F.cross_entropy in float64
on the CPU; tolerances follow test_kernel_edges.py."""
import contextlib
import copy
import math

import pytest
import torch
import torch.nn.functional as F

import pytorch_distributed_train_b200 as pdt
from pytorch_distributed_train_b200 import _C
from pytorch_distributed_train_b200.ops import functional as OF

pytestmark = pytest.mark.gpu

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
    w = torch.rand(C, device=dev(), generator=gen) + 0.25
    if kind == "some_zero":
        w[::3] = 0.0
    return w


def _targets(kind, B, C, ignore_index, gen):
    t = torch.randint(0, C, (B,), device=dev(), generator=gen)
    if kind == "half_ignored":
        t[1::2] = ignore_index
    elif kind == "all_ignored":
        t[:] = ignore_index
    return t


def _reference(x, t, w, ignore_index, reduction, eps, scale=1.0):
    """Loss and scale · d(loss)/d(logits) in float64 on the CPU, and the divisor D of the mean (None for the sum)."""
    xd = x.detach().double().cpu().requires_grad_()
    wd = None if w is None else w.double().cpu()
    tc = t.cpu()
    loss = _torch_ce(xd, tc, wd, ignore_index=ignore_index, reduction=reduction, label_smoothing=eps)
    (g,) = torch.autograd.grad(loss * scale, xd)
    counted = (tc != ignore_index) & (tc >= 0) & (tc < x.shape[1])
    D = None
    if reduction == "mean":
        D = float(counted.sum()) if wd is None else float(wd[tc[counted]].sum())
    return loss.detach(), g, D


def _assert_loss(got, ref):
    if math.isnan(ref.item()):
        assert math.isnan(got.item()), got.item()
    else:
        assert abs(got.item() - ref.item()) <= 1e-5 * abs(ref.item()) + 1e-6, (got.item(), ref.item())


def _assert_grad(got, ref, D):
    if D == 0.0:
        return   # a mean over zero total weight: the loss is NaN and so is the gradient of every counted row
    got = got.double().cpu()
    size = ref.abs().max().item()
    if size == 0.0:
        assert torch.equal(got, torch.zeros_like(got))
        return
    assert torch.allclose(got, ref, rtol=1e-5, atol=1e-6 * size), (got - ref).abs().max().item()


# ---- 1. stand-alone kernels -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("eps", [0.0, 0.1, 1.0])
@pytest.mark.parametrize("C", [1, 2, 10, 1024])
@pytest.mark.parametrize("B", [1, 7, 256, 1000])
def test_standalone_kernels_match_float64(B, C, eps, no_torch_ce):
    gen = torch.Generator(device=dev()).manual_seed(B * 7 + C)
    x = torch.randn(B, C, device=dev(), generator=gen)
    for wkind in ("none", "random", "some_zero"):
        w = _weights(wkind, C, gen)
        for reduction in ("mean", "sum"):
            for ignore_index in (-100, 3):
                for tkind in ("valid", "half_ignored", "all_ignored"):
                    # torch rejects -100 as a target when ignore_index is 3, so the ignored rows carry the ignore_index
                    t = _targets(tkind, B, C, ignore_index, gen)
                    crit = pdt.nn.CrossEntropyLoss(weight=w, ignore_index=ignore_index, reduction=reduction, label_smoothing=eps)
                    case = (wkind, reduction, ignore_index, tkind)
                    for scale in (1.0, 3.0):
                        ref_loss, ref_g, D = _reference(x, t, w, ignore_index, reduction, eps, scale)
                        xs = x.clone().requires_grad_()
                        loss = crit(xs, t)
                        (loss if scale == 1.0 else loss * scale).backward()
                        try:
                            _assert_loss(loss, ref_loss)
                            _assert_grad(xs.grad, ref_g, D)
                        except AssertionError as e:
                            raise AssertionError(f"{case} scale {scale}: {e}") from None
                    # the separate backward kernel, from the saved softmax, with an incoming gradient of 3
                    loss, probs = _C.cross_entropy_fwd(x, t, False, w, ignore_index, eps, reduction)
                    _assert_loss(loss, ref_loss)
                    assert torch.allclose(probs.double(), torch.softmax(x.double(), 1), rtol=1e-5, atol=1e-7), case
                    g = _C.cross_entropy_bwd(probs, t, torch.tensor(3.0, device=dev()), w, ignore_index, eps, reduction)
                    _assert_grad(g, ref_g, D)


def test_default_spec_is_bitwise_the_plain_kernel():
    """Explicit default options run the kernels without them: the same bits as the three-argument call."""
    x = torch.randn(100, 10, device=dev())
    t = torch.randint(0, 10, (100,), device=dev())
    t[::5] = -100
    a = _C.cross_entropy_fwd(x, t, True)
    b = _C.cross_entropy_fwd(x, t, True, None, -100, 0.0, "mean")
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_bindings_reject_bad_options():
    x = torch.randn(4, 10, device=dev())
    t = torch.randint(0, 10, (4,), device=dev())
    with pytest.raises(RuntimeError, match="reduction"):
        _C.cross_entropy_fwd(x, t, True, None, -100, 0.0, "none")
    with pytest.raises(RuntimeError, match="label_smoothing"):
        _C.cross_entropy_fwd(x, t, True, None, -100, 1.5, "mean")
    with pytest.raises(RuntimeError, match="weight"):
        _C.cross_entropy_fwd(x, t, True, torch.ones(9, device=dev()), -100, 0.0, "mean")


def test_unsupported_options_stay_on_torch():
    """reduction='none', probability targets and an out-of-range smoothing go to F.cross_entropy (which raises its own errors)."""
    x = torch.randn(6, 10, device=dev())
    t = torch.randint(0, 10, (6,), device=dev())
    got = pdt.nn.CrossEntropyLoss(reduction="none", label_smoothing=0.1)(x, t)
    assert torch.allclose(got, _torch_ce(x, t, reduction="none", label_smoothing=0.1))
    p = torch.softmax(torch.randn(6, 10, device=dev()), 1)
    assert torch.allclose(pdt.nn.CrossEntropyLoss(label_smoothing=0.1)(x, p), _torch_ce(x, p, label_smoothing=0.1))
    with pytest.raises(Exception):
        pdt.nn.CrossEntropyLoss(label_smoothing=1.5)(x, t)


# ---- 2. the forward kernel's loss rider -------------------------------------------------------------------------------------------
_SPECS = {
    "smooth": dict(label_smoothing=0.1),
    "smooth_weighted": dict(label_smoothing=0.1, weight="random"),
    "sum_zero_weights_ignore3": dict(reduction="sum", weight="some_zero", ignore_index=3),
    "ignore3": dict(ignore_index=3),
    "all_smoothing_sum": dict(label_smoothing=1.0, reduction="sum"),
}


def _criterion(name, ncls, gen):
    kw = dict(_SPECS[name])
    if "weight" in kw:
        kw["weight"] = _weights(kw["weight"], ncls, gen)
    return pdt.nn.CrossEntropyLoss(**kw)


def _spec(crit):
    return OF.ce_spec_of(crit)


@pytest.mark.parametrize("late", [False, True])
@pytest.mark.parametrize("B", ["7", "100", "sms"])
@pytest.mark.parametrize("name", list(_SPECS))
def test_forward_kernel_rider_matches_standalone_kernel(name, B, late, no_torch_ce):
    B = sms() if B == "sms" else int(B)
    gen = torch.Generator(device=dev()).manual_seed(11)
    torch.manual_seed(3)
    a = pdt.models.ConvNet(fused=True).to(dev())
    b = pdt.models.ConvNet(fused=True).to(dev())
    b.load_state_dict(a.state_dict())
    x = torch.rand(B, 1, 28, 28, device=dev(), generator=gen)
    crit = _criterion(name, 10, gen)
    t = _targets("half_ignored" if B > 1 else "valid", B, 10, crit.ignore_index, gen)
    before = _C.kernel_launch_count()
    with OF.upcoming_targets(t, loss_read_after_backward=late, spec=_spec(crit)):
        out = a(x)
    assert getattr(out, "_pdt_ce", None) is not None and out._pdt_ce[0] is t
    la = crit(out, t)
    la.backward()
    folded = _C.kernel_launch_count() - before
    before = _C.kernel_launch_count()
    lb = crit(b(x), t)
    lb.backward()
    separate = _C.kernel_launch_count() - before
    assert folded == separate - 1, (folded, separate)
    ref_loss, _, _ = _reference(out, t, crit.weight, crit.ignore_index, crit.reduction, crit.label_smoothing)
    _assert_loss(la, ref_loss)
    _assert_loss(lb, ref_loss)
    for (n1, p1), (_, p2) in zip(a.named_parameters(), b.named_parameters()):
        # softmax rounding differs in the last bit between the two kernels; the BatchNorm backward amplifies it
        scale = p2.grad.abs().max().item() + 1e-6
        assert (p1.grad - p2.grad).abs().max().item() <= 2e-3 * scale + 1e-5, (n1, (p1.grad - p2.grad).abs().max().item(), scale)


@pytest.mark.parametrize("announced,called", [
    ("default", "smooth"), ("smooth", "default"), ("smooth", "smooth_0.2"), ("smooth", "smooth_sum"), ("weighted", "weighted_copy"),
])
def test_spec_mismatch_computes_the_criterions_own_loss(announced, called, no_torch_ce):
    """The precomputed loss is used only for the same target tensor and the same options (the same weight tensor, equal scalars)."""
    gen = torch.Generator(device=dev()).manual_seed(5)
    torch.manual_seed(3)
    net = pdt.models.ConvNet(fused=True).to(dev())
    x = torch.rand(64, 1, 28, 28, device=dev(), generator=gen)
    t = torch.randint(0, 10, (64,), device=dev(), generator=gen)
    w = torch.rand(10, device=dev(), generator=gen) + 0.5
    crits = {
        "default": pdt.nn.CrossEntropyLoss(),
        "smooth": pdt.nn.CrossEntropyLoss(label_smoothing=0.1),
        "smooth_0.2": pdt.nn.CrossEntropyLoss(label_smoothing=0.2),
        "smooth_sum": pdt.nn.CrossEntropyLoss(label_smoothing=0.1, reduction="sum"),
        "weighted": pdt.nn.CrossEntropyLoss(weight=w),
        "weighted_copy": pdt.nn.CrossEntropyLoss(weight=w.clone()),
    }
    with OF.upcoming_targets(t, spec=_spec(crits[announced])):
        out = net(x)
    assert out._pdt_ce is not None
    c = crits[called]
    loss = c(out, t)
    ref_loss, _, _ = _reference(out, t, c.weight, c.ignore_index, c.reduction, c.label_smoothing)
    _assert_loss(loss, ref_loss)
    assert not hasattr(loss, "_pdt_loss_scale")   # computed by the stand-alone kernel, not taken from the forward kernel


# ---- 3. the graphed training step -------------------------------------------------------------------------------------------------
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
    g = torch.Generator(device=dev()).manual_seed(seed)
    return torch.rand(n, 1, 28, 28, device=dev(), generator=g), torch.randint(0, 10, (n,), device=dev(), generator=g)


def _rel(ours, ref):
    ours = torch.cat([o.double().reshape(-1) for o in ours])
    ref = torch.cat([r.double().reshape(-1) for r in ref])
    return (ours - ref).abs().max().item() / ref.abs().max().item()


def _smoothed_weighted():
    w = torch.rand(10, device=dev(), generator=torch.Generator(device=dev()).manual_seed(9)) + 0.25
    return pdt.nn.CrossEntropyLoss(label_smoothing=0.1, weight=w)


@pytest.mark.parametrize("optim", ["sgd", "adamw_clip"])
def test_graphed_step_with_smoothing_and_weights_follows_eager_loop(optim, no_torch_ce):
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
        # the eager loop starts where the engine's warm-up steps left the model and the optimizer
        ref = pdt.models.ConvNet().to(dev())
        ref.load_state_dict(model.state_dict())
        if optim == "sgd":
            ropt = torch.optim.SGD(ref.parameters(), 0.05, momentum=0.9, foreach=False)
        else:
            ropt = torch.optim.AdamW(ref.parameters(), 1e-3, foreach=False)
        ropt.load_state_dict(copy.deepcopy(opt.state_dict()))   # torch would otherwise share our state tensors
        for r in range(8):
            x, t = xs[r % 4]
            loss = step(x, t)
            ropt.zero_grad()
            lr_ = crit(ref(x), t)
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


@pytest.mark.parametrize("name", ["smooth", "smooth_weighted"])
def test_graphed_accumulation_with_smoothing_accumulates_in_kernel(name, no_torch_ce):
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    class ThroughAutograd(GraphedTrainStep):
        _accumulate_in_kernel = False

    k = 2
    with _one_gpu():
        gen = torch.Generator(device=dev()).manual_seed(13)
        crit = _criterion(name, 10, gen)
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
