"""SGD's three native updates against float64, and hyper-parameter schedules through every path that applies them.

The update runs in the multi-tensor kernel (``sgd_multi``, what ``SGD.step()`` launches), in the rider of the ConvNet's last
backward kernel (``SGD.ride_on_backward``, the graphed step's default on one GPU) and in the DDP reducer's fused allreduce
(``SGD.fuse_with_ddp``, world size >= 2).  Each kernel is checked against torch.optim.SGD's step in float64, one step at a time from
the values the kernel started from, at a bound derived from its roundings (``_sgd64``).  The schedule tests step a
``torch.optim.lr_scheduler`` between steps: a graphed step must replay the new learning rate, refuse a replay after any other
hyper-parameter changed, and a fused DDP step must apply the values set before its forward."""
import contextlib
import copy
import math
import types

import pytest
import torch

import pytorch_distributed_train_b200 as pdt
from mp_helpers import free_port, run_ranks

EPS = 2.0 ** -24
CONVNET = [(16, 1, 5, 5), (16,), (16,), (16,), (32, 16, 5, 5), (32,), (32,), (32,), (10, 1568), (10,)]
# momentum, dampening, weight decay, nesterov (torch allows it with a momentum and no dampening only) and maximize
CONFIGS = [dict(momentum=m, dampening=d, weight_decay=wd, nesterov=n, maximize=mx)
           for m in (0.0, 0.9) for d in (0.0, 0.5) for wd in (0.0, 1e-2) for n in (False, True) for mx in (False, True)
           if not (n and (m == 0.0 or d != 0.0))]


def _cid(c):
    return "-".join(f"{k[:4]}{v}" for k, v in c.items())


def _dev():
    return torch.device("cuda", 0)


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def _sgd64(g, p, b, lr, momentum, dampening, weight_decay, nesterov, maximize, first, absval=False):
    """torch.optim.SGD's step of one parameter in float64, with the hyper-parameters rounded to fp32 as the kernels take them and
    1 − dampening formed in fp32 as the kernels form it.  ``first``: the parameter's first momentum step (b = g).  absval: the same
    chain on magnitudes (every term added), which bounds each intermediate's magnitude for the rounding bound.

    The kernels (sgd_multi_kernel, the rider's sgd_apply, allreduce_sgd) negate for maximize (exact), then round at most five times:
    the weight-decay fma, (1 − dampening)·g, the momentum fma, the nesterov fma and the parameter fma.  Each rounding is ≤ ε = 2⁻²⁴
    of an intermediate whose magnitude, carried to the output by the same non-negative coefficients, is bounded by the magnitude
    chain; fp32 rounding of lr, momentum and weight decay adds at most three more relative errors of ε on the terms they scale
    (when the oracle takes them unrounded): |err| ≤ 9·ε·magnitude, the bound ``_check`` applies."""
    lr, mom, wd = _f32(lr), _f32(momentum), _f32(weight_decay)
    k = _f32(1.0 - _f32(dampening))
    f = (lambda t: t.abs()) if absval else (lambda t: t)
    sgn = 1.0 if absval else -1.0
    g, p = f(g), f(p)
    if maximize and not absval:
        g = -g
    if wd:
        g = g + wd * p
    if mom:
        b = g if first else mom * f(b) + k * g
        g = g + mom * b if nesterov else b
    return p + sgn * lr * g, b


def _check(what, got, ref, mag):
    err = (got.double() - ref).abs()
    bound = 9 * EPS * mag
    assert bool((err <= bound).all()), (what, (err - bound).max().item(), (err / bound.clamp_min(1e-300)).max().item())


def _flat(ts):
    return torch.cat([t.detach().double().reshape(-1) for t in ts]) if ts else torch.zeros(0, dtype=torch.float64)


def _expect_sgd(what, params, grads, p0, b0, h, first, bufs=None):
    """Every parameter (and momentum buffer) against ``_sgd64`` of its gradient from the values p0, b0 it had before the step."""
    g = _flat(grads)
    b0 = b0 if b0 is not None else torch.zeros_like(p0)
    ref_p, ref_b = _sgd64(g, p0, b0, first=first, **h)
    mag_p, mag_b = _sgd64(g, p0, b0, first=first, absval=True, **h)
    _check((what, "param"), _flat(params), ref_p, mag_p)
    if h["momentum"]:
        _check((what, "momentum buffer"), _flat(bufs), ref_b, mag_b)


def _hyper(opt, gi=0):
    g = opt.param_groups[gi]
    return {k: g[k] for k in ("lr", "momentum", "dampening", "weight_decay", "nesterov", "maximize")}


@contextlib.contextmanager
def _one_gpu():
    torch.cuda.set_device(0)
    pdt.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{free_port()}", world_size=1, rank=0)
    try:
        yield
    finally:
        pdt.destroy_process_group()


# =====================================================================================================================
# a. sgd_multi through SGD.step()
# =====================================================================================================================
def _shapes(count):
    """count parameters of sizes 1, 3, the ConvNet's, 100003, an empty one and 2²⁰ + 3 (its blocks stride 2²⁰/16384 times)."""
    if count == 1:
        return [(2 ** 20 + 3,)]
    base = [(1,), (3,)] + CONVNET + [(100003,), (0,), (2 ** 20 + 3,)]
    return [base[i % len(base)] for i in range(count)]


@pytest.mark.gpu
@pytest.mark.parametrize("count", [1, 48, 49, 100])
@pytest.mark.parametrize("lr_dev", [False, True], ids=["lr_host", "lr_dev"])
@pytest.mark.parametrize("cfg", CONFIGS, ids=[_cid(c) for c in CONFIGS])
def test_sgd_multi_matches_float64(cfg, lr_dev, count):
    """Five steps of SGD.step() over 1, 48, 49 and 100 tensors (the kernel's table holds 48): each step against float64 from the
    values it started from, one launch per 48 tensors, and the end state against torch.optim.SGD(foreach=False) in fp32."""
    from pytorch_distributed_train_b200 import _C

    gen = torch.Generator(device=_dev()).manual_seed(count * 100 + CONFIGS.index(cfg))
    shapes = _shapes(count)
    ours = [torch.randn(s, device=_dev(), generator=gen).requires_grad_() for s in shapes]
    theirs = [p.detach().clone().requires_grad_() for p in ours]
    opt = pdt.optim.SGD(ours, lr=0.05, capturable=lr_dev, **cfg)
    ref = torch.optim.SGD(theirs, lr=0.05, foreach=False, **cfg)
    h = _hyper(opt)
    for s in range(5):
        grads = [torch.randn(sh, device=_dev(), generator=gen) * 10 ** (s % 3 - 1) for sh in shapes]
        for p, q, g in zip(ours, theirs, grads):
            p.grad, q.grad = g.clone(), g.clone()
        p0 = _flat(ours)
        first = cfg["momentum"] != 0 and s == 0
        b0 = None if first or not cfg["momentum"] else _flat([opt.state[p]["momentum_buffer"] for p in ours])
        c0 = _C.kernel_launch_count()
        opt.step()
        assert _C.kernel_launch_count() - c0 == math.ceil(count / 48), "one launch per 48 tensors"
        ref.step()
        bufs = [opt.state[p]["momentum_buffer"] for p in ours] if cfg["momentum"] else None
        _expect_sgd((s, count), ours, grads, p0, b0, h, first, bufs)
    if lr_dev:
        assert opt._lr_dev[0][0].item() == _f32(0.05)
    for p, q in zip(ours, theirs):
        assert torch.allclose(p, q, atol=1e-6, rtol=1e-5), (p - q).abs().max()
        if cfg["momentum"]:
            assert torch.allclose(opt.state[p]["momentum_buffer"], ref.state[q]["momentum_buffer"], atol=1e-6, rtol=1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("lr_dev", [False, True], ids=["lr_host", "lr_dev"])
def test_sgd_multi_two_groups_with_their_own_hyper_parameters(lr_dev):
    gen = torch.Generator(device=_dev()).manual_seed(7)
    groups = [[torch.randn(s, device=_dev(), generator=gen).requires_grad_() for s in CONVNET[:5]],
              [torch.randn(s, device=_dev(), generator=gen).requires_grad_() for s in CONVNET[5:] + [(100003,)]]]
    kws = [dict(lr=0.05, momentum=0.9, dampening=0.0, weight_decay=1e-2, nesterov=True, maximize=False),
           dict(lr=0.2, momentum=0.8, dampening=0.5, weight_decay=0.0, nesterov=False, maximize=True)]
    clones = [[p.detach().clone().requires_grad_() for p in grp] for grp in groups]
    opt = pdt.optim.SGD([dict(params=grp, **kw) for grp, kw in zip(groups, kws)], lr=1.0, capturable=lr_dev)
    ref = torch.optim.SGD([dict(params=grp, **kw) for grp, kw in zip(clones, kws)], lr=1.0, foreach=False)
    for s in range(5):
        grads = [[torch.randn_like(p) for p in grp] for grp in groups]
        for grp, cl, gs in zip(groups, clones, grads):
            for p, q, g in zip(grp, cl, gs):
                p.grad, q.grad = g.clone(), g.clone()
        before = [(_flat(grp), None if s == 0 else _flat([opt.state[p]["momentum_buffer"] for p in grp])) for grp in groups]
        opt.step()
        ref.step()
        for gi, (grp, gs, (p0, b0)) in enumerate(zip(groups, grads, before)):
            _expect_sgd((s, gi), grp, gs, p0, b0, _hyper(opt, gi), s == 0, [opt.state[p]["momentum_buffer"] for p in grp])
    for p, q in zip(sum(groups, []), sum(clones, [])):
        assert torch.allclose(p, q, atol=1e-6, rtol=1e-5)
        assert torch.allclose(opt.state[p]["momentum_buffer"], ref.state[q]["momentum_buffer"], atol=1e-6, rtol=1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("dampening", [0.0, 0.5])
def test_sgd_multi_late_gradient_gets_its_own_first_step(dampening):
    """A parameter without a gradient is skipped (torch leaves it and its state alone); when its first gradient arrives, its
    momentum buffer starts at that gradient (no dampening) while the others take an ordinary step: two launches, as torch
    decides the first step per parameter."""
    from pytorch_distributed_train_b200 import _C

    gen = torch.Generator(device=_dev()).manual_seed(8)
    ours = [torch.randn(s, device=_dev(), generator=gen).requires_grad_() for s in CONVNET]
    theirs = [p.detach().clone().requires_grad_() for p in ours]
    late = (4, 9)
    kw = dict(lr=0.05, momentum=0.9, dampening=dampening, weight_decay=1e-2)
    opt = pdt.optim.SGD(ours, **kw)
    ref = torch.optim.SGD(theirs, foreach=False, **kw)
    for s in range(5):
        idx = [i for i in range(len(ours)) if s >= 2 or i not in late]
        frozen = [ours[i].detach().clone() for i in late]
        for i in range(len(ours)):
            g = torch.randn_like(ours[i]) if i in idx else None
            ours[i].grad, theirs[i].grad = g, None if g is None else g.clone()
        before = {i: (ours[i].detach().double().reshape(-1), None if "momentum_buffer" not in opt.state[ours[i]] or
                      opt.state[ours[i]]["momentum_buffer"] is None else _flat([opt.state[ours[i]]["momentum_buffer"]])) for i in idx}
        c0 = _C.kernel_launch_count()
        opt.step()
        assert _C.kernel_launch_count() - c0 == (2 if s == 2 else 1), s
        ref.step()
        for i in idx:
            p0, b0 = before[i]
            _expect_sgd((s, i), [ours[i]], [ours[i].grad], p0, b0, _hyper(opt), b0 is None, [opt.state[ours[i]]["momentum_buffer"]])
        if s < 2:
            for i, f in zip(late, frozen):
                assert torch.equal(ours[i].detach(), f) and opt.state[ours[i]].get("momentum_buffer") is None
    for p, q in zip(ours, theirs):
        assert torch.allclose(p, q, atol=1e-6, rtol=1e-5)
        assert torch.allclose(opt.state[p]["momentum_buffer"], ref.state[q]["momentum_buffer"], atol=1e-6, rtol=1e-5)


# =====================================================================================================================
# b. the rider of the last backward kernel
# =====================================================================================================================
def _batch(seed, rows=100):
    g = torch.Generator(device=_dev()).manual_seed(seed)
    return torch.rand(rows, 1, 28, 28, device=_dev(), generator=g), torch.randint(0, 10, (rows,), device=_dev(), generator=g)


def _state(model, opt):
    params = list(model.parameters())
    bufs = [opt.state[p].get("momentum_buffer") for p in params]
    return params, _flat(params), None if any(b is None for b in bufs) else _flat(bufs)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain", "clip2", "clipinf", "accumulate2"])
@pytest.mark.parametrize("cfg", CONFIGS, ids=[_cid(c) for c in CONFIGS])
def test_rider_matches_float64_of_its_own_gradients(cfg, mode):
    """The last backward kernel's update of all ten ConvNet parameters against float64 of the gradients it stored (clipped, or
    accumulated over two micro-batches, where it does that first), with the lr in a device scalar.  The bn2 and fc parameters are
    updated in the shadow of the kernel's first grid barrier from gradients an earlier kernel wrote: the value a thread updates
    with must be the one in .grad."""
    from pytorch_distributed_train_b200.engine import GraphedTrainStep
    from pytorch_distributed_train_b200.ops import functional as OF

    torch.manual_seed(3)
    model = pdt.models.ConvNet(fused=True).to(_dev())
    opt = pdt.optim.SGD(model.parameters(), 0.05, capturable=True, **cfg)
    crit = pdt.nn.CrossEntropyLoss()
    h = _hyper(opt)
    if mode == "accumulate2":
        with _one_gpu():
            x, t = _batch(0, 200)
            step = GraphedTrainStep(pdt.DistributedDataParallel(model, device_ids=[0]), crit, opt, (x, t), warmup=2,
                                    accumulation_steps=2, double_buffer_inputs=False)
            assert step._riding and step.accumulates_in_kernel and step.kernels_per_replay == 6, step.kernels_per_replay
            for s in range(3):
                params, p0, b0 = _state(model, opt)
                x, t = _batch(10 + s, 200)
                step(x, t)
                torch.cuda.synchronize()
                _expect_sgd(s, params, [p.grad for p in params], p0, b0, h, False, [opt.state[p].get("momentum_buffer") for p in params])
            opt.stop_riding()
        return
    clip = None
    if mode != "plain":
        norm_out = torch.zeros(1, device=_dev())
        clip = (0.05, 2.0 if mode == "clip2" else math.inf, norm_out)
    assert opt.ride_on_backward(model, clip=clip)
    try:
        for s in range(3):
            params, p0, b0 = _state(model, opt)
            x, t = _batch(s)
            opt.zero_grad()
            loss = crit(model(x), t)
            with OF.sgd_rider_enabled():
                loss.backward()
            assert opt._rode
            opt.step()
            torch.cuda.synchronize()
            if clip is not None:
                assert norm_out.item() > clip[0], "the gradients must have been clipped"
            _expect_sgd(s, params, [p.grad for p in params], p0, b0, h, cfg["momentum"] != 0 and s == 0,
                        [opt.state[p].get("momentum_buffer") for p in params])
    finally:
        opt.stop_riding()


# =====================================================================================================================
# c. learning-rate schedules through GraphedTrainStep
# =====================================================================================================================
OPTS = {"sgd": (pdt.optim.SGD, dict(lr=0.05)), "sgd_momentum": (pdt.optim.SGD, dict(lr=0.05, momentum=0.9, weight_decay=1e-3)),
        "adamw": (pdt.optim.AdamW, dict(lr=1e-3))}


def _rel(ours, ref):
    """bench.py's verification metric: max |ours − reference| / max |reference| over the flat vector."""
    return (_flat(ours) - _flat(ref)).abs().max().item() / _flat(ref).abs().max().item()


@pytest.mark.gpu
# the replays run the update, never optimizer.step() itself, which torch's schedulers expect to see before their own step
@pytest.mark.filterwarnings("ignore:Detected call of `lr_scheduler.step\\(\\)` before `optimizer.step\\(\\)`")
@pytest.mark.parametrize("path", ["rider", "unfused", "clip_unfused"])
@pytest.mark.parametrize("capturable", [False, True])
@pytest.mark.parametrize("name", list(OPTS))
def test_graphed_step_follows_a_learning_rate_schedule(name, capturable, path, monkeypatch):
    """A LambdaLR that alternates lr between its value and 0, stepped between replays: a replay at lr 0 leaves every parameter
    bitwise unchanged (p − 0·u is p), a replay at lr > 0 of SGD matches float64 of that replay's gradients, and the run follows an
    eager loop of the same model and optimizer through the same schedule."""
    from pytorch_distributed_train_b200.engine import GraphedTrainStep
    from pytorch_distributed_train_b200.nn.utils import clip_grad_norm_

    if path != "rider":
        monkeypatch.setenv("PDT_SGD_RIDER", "0")
    cls, kw = OPTS[name]
    clip = 0.5 if path.startswith("clip") else None
    with _one_gpu():
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(_dev())
        opt = cls(model.parameters(), capturable=capturable, **kw)
        crit = pdt.nn.CrossEntropyLoss()
        xs = [_batch(20 + i) for i in range(4)]
        step = GraphedTrainStep(pdt.DistributedDataParallel(model, device_ids=[0]), crit, opt, xs[0], warmup=3, max_grad_norm=clip,
                                double_buffer_inputs=False)
        assert step._riding == (path == "rider")
        assert opt.param_groups[0]["capturable"] == capturable, "the user's param_groups stay as they were"
        # the eager reference starts where the warm-up steps left the model and the optimizer
        ref = pdt.models.ConvNet().to(_dev())
        ref.load_state_dict(model.state_dict())
        ropt = cls(ref.parameters(), capturable=capturable, **kw)
        ropt.load_state_dict(copy.deepcopy(opt.state_dict()))
        sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda e: 0.0 if e % 2 else 1.0)
        rsched = torch.optim.lr_scheduler.LambdaLR(ropt, lambda e: 0.0 if e % 2 else 1.0)
        for i in range(8):
            lr = opt.param_groups[0]["lr"]
            assert lr == (0.0 if i % 2 else kw["lr"])
            params, p0, b0 = _state(model, opt)
            step(*xs[i % 4], inputs_ready=True)
            torch.cuda.synchronize()
            if lr == 0.0:
                assert torch.equal(_flat(params), p0), (i, "a replay at lr 0 changed the parameters")
            elif cls is pdt.optim.SGD:
                _expect_sgd(i, params, [p.grad for p in params], p0, b0, _hyper(opt), False,
                            [opt.state[p].get("momentum_buffer") for p in params])
            ropt.zero_grad()
            crit(ref(xs[i % 4][0]), xs[i % 4][1]).backward()
            if clip is not None:
                clip_grad_norm_(list(ref.parameters()), clip)
            ropt.step()
            sched.step()
            rsched.step()
        # bench.py's tolerance; Adam scales the rounding noise of the two convolution biases (they feed a BatchNorm) up to
        # full-size steps, so they are left out for AdamW as in test_adam.py
        skip = ("layer1.0.bias", "layer2.0.bias") if name == "adamw" else ()
        keep = [(p, q) for (n, p), q in zip(model.named_parameters(), ref.parameters()) if n not in skip]
        err = _rel([p for p, _ in keep], [q for _, q in keep])
        assert err < 2e-2, err
        opt.stop_riding()


# =====================================================================================================================
# d. schedules of other hyper-parameters: OneCycleLR(cycle_momentum=True)
# =====================================================================================================================
@pytest.mark.gpu
def test_eager_sgd_follows_one_cycle_momentum_in_float64():
    gen = torch.Generator(device=_dev()).manual_seed(11)
    ours = [torch.randn(s, device=_dev(), generator=gen).requires_grad_() for s in CONVNET]
    theirs = [p.detach().double().clone().requires_grad_() for p in ours]
    opt = pdt.optim.SGD(ours, lr=0.05, momentum=0.9, weight_decay=1e-3)
    ref = torch.optim.SGD(theirs, lr=0.05, momentum=0.9, weight_decay=1e-3, foreach=False)
    scheds = [torch.optim.lr_scheduler.OneCycleLR(o, max_lr=0.1, total_steps=8, cycle_momentum=True) for o in (opt, ref)]
    seen = set()
    for s in range(8):
        assert _hyper(opt) == _hyper(ref), s
        seen.add(opt.param_groups[0]["momentum"])
        grads = [torch.randn_like(p) for p in ours]
        p0 = _flat(ours)
        b0 = None if s == 0 else _flat([opt.state[p]["momentum_buffer"] for p in ours])
        with torch.no_grad():   # torch's float64 step from our values: the oracle of this step
            for p, q, g in zip(ours, theirs, grads):
                q.copy_(p)
                q.grad = g.double()
                if s:
                    ref.state[q]["momentum_buffer"].copy_(opt.state[p]["momentum_buffer"])
        for p, g in zip(ours, grads):
            p.grad = g
        opt.step()
        ref.step()
        mag_p, mag_b = _sgd64(_flat(grads), p0, b0 if b0 is not None else torch.zeros_like(p0), first=s == 0, absval=True, **_hyper(opt))
        _check((s, "param"), _flat(ours), _flat(theirs), mag_p)
        _check((s, "momentum buffer"), _flat([opt.state[p]["momentum_buffer"] for p in ours]),
               _flat([ref.state[q]["momentum_buffer"] for q in theirs]), mag_b)
        for sc in scheds:
            sc.step()
    assert len(seen) >= 4, "the schedule must have moved the momentum"


@pytest.mark.gpu
def test_eager_adamw_follows_one_cycle_betas_in_float64():
    gen = torch.Generator(device=_dev()).manual_seed(12)
    ours = [torch.randn(s, device=_dev(), generator=gen).requires_grad_() for s in CONVNET]
    theirs = [p.detach().double().clone().requires_grad_() for p in ours]
    opt = pdt.optim.AdamW(ours, lr=1e-3)
    ref = torch.optim.AdamW(theirs, lr=1e-3, foreach=False)
    scheds = [torch.optim.lr_scheduler.OneCycleLR(o, max_lr=1e-2, total_steps=8, cycle_momentum=True) for o in (opt, ref)]
    seen = set()
    for s in range(8):
        assert opt.param_groups[0]["betas"] == ref.param_groups[0]["betas"] and opt.param_groups[0]["lr"] == ref.param_groups[0]["lr"]
        seen.add(opt.param_groups[0]["betas"][0])
        grads = [torch.randn_like(p) for p in ours]
        p0 = [p.detach().double().clone() for p in ours]
        with torch.no_grad():   # torch's float64 step from our values: the oracle of this step
            for p, q, g in zip(ours, theirs, grads):
                q.copy_(p)
                q.grad = g.double()
                if s:
                    st, rt = opt.state[p], ref.state[q]
                    rt["exp_avg"].copy_(st["exp_avg"])
                    rt["exp_avg_sq"].copy_(st["exp_avg_sq"])
                    rt["step"].fill_(st["step"].item())
        for p, g in zip(ours, grads):
            p.grad = g
        opt.step()
        ref.step()
        # test_adam.py's float64 tolerance: relative to the largest magnitude the value was formed from
        for i, (p, q, g) in enumerate(zip(ours, theirs, grads)):
            st, rt = opt.state[p], ref.state[q]
            assert st["step"].item() == rt["step"].item() == s + 1
            for name, x, y, scale in (("p", p, q, p0[i].abs()), ("exp_avg", st["exp_avg"], rt["exp_avg"], g.double().abs()),
                                      ("exp_avg_sq", st["exp_avg_sq"], rt["exp_avg_sq"], rt["exp_avg_sq"].abs())):
                err = (x.double() - y.detach()).abs()
                assert bool((err <= 1e-5 * torch.maximum(y.detach().abs(), scale) + 1e-7).all()), (s, i, name, err.max().item())
        for sc in scheds:
            sc.step()
    assert len(seen) >= 4, "the schedule must have moved beta1"


@pytest.mark.gpu
@pytest.mark.parametrize("name,key", [("sgd_momentum", "momentum"), ("adamw", "betas")])
def test_graphed_step_refuses_a_replay_after_one_cycle_moved_momentum(name, key):
    """OneCycleLR(cycle_momentum=True) changes the momentum (SGD) or betas[0] (AdamW) on every step.  A captured step bakes them into
    its kernels, so the first replay after a change must raise, naming the hyper-parameter, before it runs anything."""
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    cls, kw = OPTS[name]
    with _one_gpu():
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(_dev())
        opt = cls(model.parameters(), **kw)
        sched = torch.optim.lr_scheduler.OneCycleLR(opt, max_lr=2 * kw["lr"], total_steps=10, cycle_momentum=True)
        xs = [_batch(30 + i) for i in range(2)]
        step = GraphedTrainStep(pdt.DistributedDataParallel(model, device_ids=[0]), pdt.nn.CrossEntropyLoss(), opt, xs[0], warmup=3)
        step(*xs[1], inputs_ready=True)   # the values the step was captured with: replays
        sched.step()                      # lr and the momentum move; bookkeeping keys (initial_lr, max_momentum, ...) stay
        torch.cuda.synchronize()
        params, p0, _ = _state(model, opt)
        replays = step.replays
        with pytest.raises(RuntimeError, match=f"'{key}'"):
            step(*xs[0], inputs_ready=True)
        torch.cuda.synchronize()
        assert step.replays == replays and torch.equal(_flat(params), p0), "a refused replay must not run"


def _perturbed(v):
    if isinstance(v, bool):
        return not v
    if isinstance(v, tuple):
        return tuple(x / 2 for x in v)
    return None if v is None else v / 2 + 0.25


@pytest.mark.parametrize("cls", [pdt.optim.SGD, pdt.optim.Adam, pdt.optim.AdamW])
def test_replay_check_covers_every_key_the_update_reads(cls):
    """A graphed step refuses a replay when one of _FIXED_KEYS changed (one tuple comparison per replay): they must be exactly the
    group keys besides lr that change what _hyper hands the kernels."""
    opt = cls([torch.zeros(3, requires_grad=True)], lr=0.1)
    group = opt.param_groups[0]
    base = opt._hyper(0, group, torch.device("cpu"))
    reads = set()
    for key in [k for k in group if k not in ("params", "lr")]:
        old = group[key]
        group[key] = _perturbed(old)
        if opt._hyper(0, group, torch.device("cpu")) != base:
            reads.add(key)
        group[key] = old
    assert reads == set(cls._FIXED_KEYS), (reads, cls._FIXED_KEYS)
    opt._record_captured_hyper()
    opt.sync_lr()
    for key in cls._FIXED_KEYS:
        old = group[key]
        group[key] = _perturbed(old)
        with pytest.raises(RuntimeError, match=f"'{key}' of param_groups\\[0\\]"):
            opt.sync_lr()
        group[key] = old
    opt.sync_lr()


# =====================================================================================================================
# e. the update fused into DDP's gradient reduction
# =====================================================================================================================
class _RecordingReducer:
    """Stands in for the native reducer: records what set_fused_sgd installs."""

    def __init__(self):
        self.armed = []

    @property
    def fused_sgd(self):
        return bool(self.armed)

    def prepare_for_forward(self):
        pass

    def set_fused_sgd(self, param_flat, momentum_flat=None, **hyper):
        self.armed.append(hyper)


class _FusableDDP:
    """Just enough of pdt.DistributedDataParallel for SGD.fuse_with_ddp, with DDP's own forward prologue."""

    _pre_forward = pdt.DistributedDataParallel._pre_forward

    def __init__(self, params):
        self._params = params
        self._param_offsets = [0]
        for p in params[:-1]:
            self._param_offsets.append(self._param_offsets[-1] + p.numel())
        self.param_arena = torch.zeros(sum(p.numel() for p in params))
        self.process_group = types.SimpleNamespace(size=lambda: 2)
        self.reducer = _RecordingReducer()
        self.require_backward_grad_sync = True
        self._join_active = False
        self.broadcast_buffers = False
        self.device_ids = None
        self.settled = False   # the reducer settles its bucket layout after the first iteration

    def _maybe_rebuild_buckets(self):
        pass

    def enable_optimizer_fusion(self):
        return self.settled

    def tail_broadcast_buffer(self):
        return None


def test_fused_ddp_arms_the_hyper_parameters_set_before_the_forward():
    """The update the reducer applies during a backward must use the hyper-parameters in param_groups when that iteration's
    forward started: a scheduler stepped after step() takes effect in the next iteration (not one late), and so does a change
    of momentum, dampening or weight decay.  A change between forward and backward waits for the next forward."""
    params = [torch.randn(5, requires_grad=True), torch.randn(3, requires_grad=True)]
    ddp = _FusableDDP(params)
    opt = pdt.optim.SGD(params, lr=0.1, momentum=0.9).fuse_with_ddp(ddp)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda e: 0.5 ** e)
    keys = ("lr", "momentum", "dampening", "weight_decay", "nesterov")
    for it in range(8):
        if it == 4:
            opt.param_groups[0]["momentum"] = 0.5
        if it == 5:
            opt.param_groups[0].update(dampening=0.25, weight_decay=1e-2)
        want = {k: opt.param_groups[0][k] for k in keys}
        ddp._pre_forward((), {})
        if it == 6:
            opt.param_groups[0]["lr"] = 123.0   # between forward and backward: not this iteration's
        if opt._fused_active:   # the backward: the reducer applies what is armed now
            got = ddp.reducer.armed[-1]
            assert {k: got[k] for k in keys} == want, (it, got, want)
            assert got["first_step"] is False
        for p in params:
            p.grad = torch.ones_like(p)
        opt.step()
        ddp.settled = True
        if it == 6:
            ddp._pre_forward((), {})
            assert ddp.reducer.armed[-1]["lr"] == 123.0, "picked up by the next forward"
            opt.param_groups[0]["lr"] = want["lr"]
        sched.step()
    assert opt._fused_active and len(ddp.reducer.armed) >= 6


def _ddp_schedule(rank, world, fused):
    """Eager DDP training with a LambdaLR that sets lr to 0 every third step and a momentum change, fused or not: the parameters
    after every step."""
    dev = torch.device("cuda", rank)
    torch.manual_seed(0)
    model = pdt.models.ConvNet().to(dev)
    opt = pdt.optim.SGD(model.parameters(), 0.05, momentum=0.9, weight_decay=1e-3)
    ddp = pdt.DistributedDataParallel(model, device_ids=[rank])
    if fused:
        opt.fuse_with_ddp(ddp)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda e: 0.0 if e % 3 == 2 else 1.0)
    crit = pdt.nn.CrossEntropyLoss()
    out = []
    for s in range(12):
        if s == 7:
            opt.param_groups[0]["momentum"] = 0.5
        g = torch.Generator().manual_seed(1000 * s + rank)
        x, y = torch.rand(100, 1, 28, 28, generator=g).to(dev), torch.randint(0, 10, (100,), generator=g).to(dev)
        loss = crit(ddp(x), y)
        opt.zero_grad()
        loss.backward()
        opt.step()
        sched.step()
        torch.cuda.synchronize()
        out.append(torch.cat([p.detach().reshape(-1) for p in ddp.parameters()]).cpu())
    return bool(opt._fused_active), out


@pytest.mark.gpu
@pytest.mark.multigpu
def test_fused_ddp_follows_a_schedule_step_for_step():
    world = 2
    plain = run_ranks(_ddp_schedule, world, False, backend="nccl")
    fused = run_ranks(_ddp_schedule, world, True, backend="nccl")
    for (pa, a), (fa, b) in zip(plain, fused):
        assert not pa and fa
        prev = None
        for s, (x, y) in enumerate(zip(a, b)):
            # the two paths differ by FMA ordering only; TF32 operands in the convolutions amplify it (test_fused_allreduce_sgd)
            scale = x.abs().max().item()
            assert (x - y).abs().max().item() < 2e-3 * scale, (s, (x - y).abs().max().item(), scale)
            if s >= 3 and s % 3 == 2:   # fused from step 2 on; lr 0 in this step: p − 0·u is p
                assert torch.equal(y, prev), (s, "the fused update of an lr-0 step changed the parameters")
            prev = y
    assert torch.equal(fused[0][1][-1], fused[-1][1][-1])   # ranks bit-identical
