"""pdt.optim.RMSprop and pdt.optim.Adagrad: torch's constructors, state and reference arithmetic on the CPU; on the GPU the
multi-tensor kernels (rmsprop_multi_kernel, adagrad_multi_kernel) and the riders of the ConvNet's last backward kernel against
float64, one step at a time from the values the step started from, at bounds derived from their roundings (``_rmsprop64``,
``_adagrad64``); GraphedTrainStep with both, under a learning-rate schedule and, for Adagrad, a learning-rate decay that has to
advance from replay to replay."""
import contextlib
import copy
import math
import os
import subprocess
import sys

import pytest
import torch

import pytorch_distributed_train_b200 as pdt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = 2.0 ** -24
CONVNET = [(16, 1, 5, 5), (16,), (16,), (16,), (32, 16, 5, 5), (32,), (32,), (32,), (10, 1568), (10,)]
# the ConvNet's biases of the two convolutions feed a BatchNorm: their gradient is rounding noise, which RMSprop and Adagrad
# scale up to full-size steps, so comparisons of two different gradient paths leave them out (as test_adam.py does)
NOISE = ("layer1.0.bias", "layer2.0.bias")
PAIRS = [(pdt.optim.RMSprop, torch.optim.RMSprop), (pdt.optim.Adagrad, torch.optim.Adagrad)]
RMSPROP_CONFIGS = {"plain": {}, "wd": dict(weight_decay=1e-2), "momentum": dict(momentum=0.9), "centered": dict(centered=True),
                   "centered_momentum": dict(centered=True, momentum=0.9), "maximize": dict(maximize=True)}
ADAGRAD_CONFIGS = {"plain": {}, "lr_decay": dict(lr_decay=0.1), "wd": dict(weight_decay=1e-2),
                   "initial_accumulator_value": dict(initial_accumulator_value=0.5), "maximize": dict(maximize=True)}


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def _flat(ts):
    return torch.cat([t.detach().double().reshape(-1) for t in ts]) if ts else torch.zeros(0, dtype=torch.float64)


# =====================================================================================================================
# float64 oracles with their rounding bounds
# =====================================================================================================================
def _sqrt_err(x, e):
    """Error bound of sqrt(x) when x carries an error of at most e: e / (2·sqrt(x)) to first order, and never more than sqrt(e)."""
    return torch.minimum(e / (2 * x.clamp_min(1e-300).sqrt()), e.sqrt())


def _rmsprop64(g, p, sq, ga, buf, lr, alpha, eps, weight_decay, momentum, maximize, centered):
    """torch.optim.RMSprop's step of flat float64 vectors from the values p, sq, ga (centered), buf (momentum > 0) the kernel started
    from, with the hyper-parameters rounded to fp32 as the kernels take them (1 − α formed in double, then rounded).  Returns
    (reference, bound) pairs for p, square_avg, grad_avg and momentum_buffer.

    The kernels (rmsprop_multi_kernel, the rider's rmsprop_apply) negate for maximize (exact), then round once in each of: the
    weight-decay fma g' = wd·p + g; (1 − α)·g', α·sq and the fma sq' = (1 − α)g'·g' + α·sq; centered: g' − ga, the lerp fma
    ga' = (1 − α)(g' − ga) + ga and the fma var = sq' − ga'² (exact product, one rounding, so ≤ ε·|var|); sqrt (correctly rounded);
    + eps; the division u = g'/avg; momentum: the fma buf' = m·buf + u; the fma p' = p − lr·(buf' or u).  Each rounding is ≤ ε = 2⁻²⁴
    of its result, and the errors of the inputs of each operation are carried through it to first order (through sqrt by
    _sqrt_err, through the division by |δg'|/avg + |u|·δavg/(avg − δavg)).  var's error is bounded relative to sq' + ga'² (the
    magnitudes it is formed from), not to var.  The bound is twice the first-order sum, which covers the second-order terms."""
    lr, alpha, oma, eps, wd, mom = _f32(lr), _f32(alpha), _f32(1.0 - alpha), _f32(eps), _f32(weight_decay), _f32(momentum)
    g = -g if maximize else g
    e_g = torch.zeros_like(g)
    if wd:
        e_g = EPS * (g + wd * p).abs()
        g = g + wd * p
    sq1 = alpha * sq + oma * g * g
    e_sq = EPS * (2 * oma * g * g + alpha * sq + sq1) + 2 * oma * g.abs() * e_g
    var, e_var, ga1, e_ga = sq1, e_sq, None, None
    if centered:
        d = g - ga
        ga1 = ga + oma * d
        e_ga = EPS * (oma * d.abs() + ga1.abs()) + oma * e_g
        var = sq1 - ga1 * ga1
        e_var = EPS * var.abs() + e_sq + 2 * ga1.abs() * e_ga
    root = var.clamp_min(0).sqrt()
    avg = root + eps
    e_avg = _sqrt_err(var.clamp_min(0), e_var) + EPS * root + EPS * avg
    u = g / avg
    e_u = EPS * u.abs() + e_g / avg + u.abs() * e_avg / (avg - e_avg)
    step, e_step, buf1, e_buf = u, e_u, None, None
    if mom > 0:
        buf1 = mom * buf + u
        e_buf = EPS * buf1.abs() + e_u
        step, e_step = buf1, e_buf
    p1 = p - lr * step
    e_p = EPS * p1.abs() + lr * e_step
    return (p1, 2 * e_p), (sq1, 2 * e_sq), (ga1, None if e_ga is None else 2 * e_ga), (buf1, None if e_buf is None else 2 * e_buf)


def _adagrad64(g, p, s, step, lr, lr_decay, eps, weight_decay, maximize):
    """torch.optim.Adagrad's step of flat float64 vectors from the values p, s (sum) and the step count `step` the kernel started
    from: clr = lr / (1 + step·lr_decay) with lr as the kernel reads it (the host's double, or fp32 from the device scalar), eps and
    the weight decay rounded to fp32.  Returns (reference, bound) pairs for p and sum.

    The kernels (adagrad_multi_kernel, the rider's adagrad_apply) negate for maximize (exact), then round once in each of: clr to
    fp32; the weight-decay fma g' = wd·p + g; the fma sum' = g'·g' + sum; sqrt; + eps; the division u = g'/std; the fma p' = p − clr·u.
    Each rounding is ≤ ε = 2⁻²⁴ of its result, input errors are carried to first order as in _rmsprop64, and the bound is twice the
    first-order sum."""
    eps, wd = _f32(eps), _f32(weight_decay)
    clr = lr / (1.0 + step * lr_decay)
    g = -g if maximize else g
    e_g = torch.zeros_like(g)
    if wd:
        e_g = EPS * (g + wd * p).abs()
        g = g + wd * p
    s1 = s + g * g
    e_s = EPS * s1 + 2 * g.abs() * e_g
    root = s1.sqrt()
    std = root + eps
    e_std = _sqrt_err(s1, e_s) + EPS * root + EPS * std
    u = g / std
    e_u = EPS * u.abs() + e_g / std + u.abs() * e_std / (std - e_std)
    p1 = p - clr * u
    e_p = EPS * p1.abs() + clr * e_u + EPS * clr * u.abs()
    return (p1, 2 * e_p), (s1, 2 * e_s)


def _check(what, got, ref_bound):
    ref, bound = ref_bound
    err = (got.double() - ref).abs()
    ok = err <= bound
    assert bool(ok.all()), (what, int((~ok).sum()), (err - bound).max().item(), (err / bound.clamp_min(1e-300)).max().item())


def _close(x, y):
    """fp32 agreement of two runs of the same steps, relative to the tensor's largest magnitude: a momentum buffer or grad_avg sums
    terms of both signs, so an element can be far smaller than the terms (and their roundings) it was formed from."""
    scale = float(y[~torch.isnan(y)].abs().max()) if y.numel() else 0.0
    return torch.allclose(x, y, rtol=1e-5, atol=1e-7 + 1e-6 * scale, equal_nan=True)


def _state_of(opt, params, key):
    return _flat([opt.state[p][key] for p in params]) if all(key in opt.state[p] for p in params) else None


def _snapshot(opt, params):
    """The flat values an RMSprop or Adagrad step starts from: p and every state tensor, and the first step count."""
    snap = {"p": _flat(params)}
    for key in ("square_avg", "grad_avg", "momentum_buffer", "sum"):
        snap[key] = _state_of(opt, params, key)
    snap["step"] = float(opt.state[params[0]]["step"]) if "step" in opt.state[params[0]] else 0.0
    return snap


def _lr_read(opt, group):
    """The learning rate as the kernels read it: fp32 from the device scalar when the optimizer keeps one, else the host's value."""
    return _f32(group["lr"]) if (group.get("capturable") or opt._lr_on_device) else group["lr"]


def _expect(what, opt, params, grads, snap):
    """Every parameter and state tensor of one RMSprop or Adagrad step against float64 from the snapshot the step started from."""
    g, grp = _flat(grads), opt.param_groups[0]
    zeros = torch.zeros_like(snap["p"])
    if isinstance(opt, pdt.optim.RMSprop):
        rp, rsq, rga, rbuf = _rmsprop64(g, snap["p"], snap["square_avg"] if snap["square_avg"] is not None else zeros,
                                        snap["grad_avg"] if snap["grad_avg"] is not None else zeros,
                                        snap["momentum_buffer"] if snap["momentum_buffer"] is not None else zeros,
                                        grp["lr"], grp["alpha"], grp["eps"], grp["weight_decay"], grp["momentum"], grp["maximize"],
                                        grp["centered"])
        _check((what, "square_avg"), _state_of(opt, params, "square_avg"), rsq)
        if grp["centered"]:
            _check((what, "grad_avg"), _state_of(opt, params, "grad_avg"), rga)
        if grp["momentum"] > 0:
            _check((what, "momentum_buffer"), _state_of(opt, params, "momentum_buffer"), rbuf)
    else:
        rp, rs = _adagrad64(g, snap["p"], snap["sum"], snap["step"], _lr_read(opt, grp), grp["lr_decay"], grp["eps"],
                            grp["weight_decay"], grp["maximize"])
        _check((what, "sum"), _state_of(opt, params, "sum"), rs)
    _check((what, "param"), _flat(params), rp)
    assert all(float(opt.state[p]["step"]) == snap["step"] + 1 for p in params), (what, "step")


# =====================================================================================================================
# CPU
# =====================================================================================================================
@pytest.mark.parametrize("ours,theirs", PAIRS, ids=["rmsprop", "adagrad"])
def test_defaults_match_torch(ours, theirs):
    p = [torch.zeros(3, requires_grad=True)]
    a, b = ours(p), theirs([torch.zeros(3, requires_grad=True)])
    assert a.defaults == b.defaults
    ga, gb = dict(a.param_groups[0]), dict(b.param_groups[0])
    ga.pop("params"), gb.pop("params")
    assert ga == gb


BAD = {pdt.optim.RMSprop: [dict(lr=-1.0), dict(eps=-1e-8), dict(momentum=-0.5), dict(weight_decay=-1.0), dict(alpha=-0.1),
                           dict(lr=torch.tensor([0.1, 0.2]))],
       pdt.optim.Adagrad: [dict(lr=-1.0), dict(lr_decay=-0.1), dict(weight_decay=-1.0), dict(initial_accumulator_value=-1.0),
                           dict(eps=-1e-10), dict(lr=torch.tensor([0.1, 0.2]))]}


@pytest.mark.parametrize("ours,theirs", PAIRS, ids=["rmsprop", "adagrad"])
def test_constructor_errors_match_torch(ours, theirs):
    for kw in BAD[ours]:
        with pytest.raises(ValueError) as mine:
            ours([torch.zeros(2, requires_grad=True)], **kw)
        with pytest.raises(ValueError) as ref:
            theirs([torch.zeros(2, requires_grad=True)], **kw)
        assert str(mine.value) == str(ref.value), kw
    if ours is pdt.optim.Adagrad:
        for kw in (dict(fused=True, differentiable=True), dict(fused=True, foreach=True)):
            with pytest.raises(RuntimeError) as mine:
                ours([torch.zeros(2, requires_grad=True)], **kw)
            with pytest.raises(RuntimeError) as ref:
                theirs([torch.zeros(2, requires_grad=True)], **kw)
            assert str(mine.value) == str(ref.value), kw


def _cpu_params(dtype=torch.float32, complex_too=False, seed=0):
    g = torch.Generator().manual_seed(seed)
    ps = [torch.randn(s, generator=g, dtype=dtype).requires_grad_() for s in [(5, 3), (7,), (1,)]]
    if complex_too:
        ps.append(torch.randn(4, generator=g, dtype=torch.complex64).requires_grad_())
    return ps


@pytest.mark.parametrize("cfg", list(RMSPROP_CONFIGS), ids=list(RMSPROP_CONFIGS))
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_rmsprop_reference_step_matches_torch_bit_for_bit(cfg, dtype):
    """CPU parameters (and a complex one) take torch's single-tensor arithmetic: five steps equal torch.optim.RMSprop(foreach=False)
    bit for bit, state keys included."""
    kw = RMSPROP_CONFIGS[cfg]
    pa = _cpu_params(dtype, complex_too=True)
    pb = [p.detach().clone().requires_grad_() for p in pa]
    a, b = pdt.optim.RMSprop(pa, lr=1e-2, **kw), torch.optim.RMSprop(pb, lr=1e-2, foreach=False, **kw)
    gen = torch.Generator().manual_seed(1)
    for _ in range(5):
        for p, q in zip(pa, pb):
            p.grad = torch.randn(p.shape, generator=gen, dtype=p.dtype)
            q.grad = p.grad.clone()
        a.step()
        b.step()
    want = {"step", "square_avg"} | ({"momentum_buffer"} if kw.get("momentum", 0) > 0 else set()) | ({"grad_avg"} if kw.get("centered") else set())
    for p, q in zip(pa, pb):
        assert set(a.state[p]) == set(b.state[q]) == want
        assert torch.equal(p, q)
        for k in want:
            assert torch.equal(a.state[p][k], b.state[q][k]), k


@pytest.mark.parametrize("cfg", list(ADAGRAD_CONFIGS), ids=list(ADAGRAD_CONFIGS))
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_adagrad_reference_step_matches_torch_bit_for_bit(cfg, dtype):
    kw = ADAGRAD_CONFIGS[cfg]
    pa = _cpu_params(dtype, complex_too=True)
    pb = [p.detach().clone().requires_grad_() for p in pa]
    a, b = pdt.optim.Adagrad(pa, lr=1e-2, **kw), torch.optim.Adagrad(pb, lr=1e-2, foreach=False, **kw)
    gen = torch.Generator().manual_seed(1)
    for _ in range(5):
        for p, q in zip(pa, pb):
            p.grad = torch.randn(p.shape, generator=gen, dtype=p.dtype)
            q.grad = p.grad.clone()
        a.step()
        b.step()
    for p, q in zip(pa, pb):
        assert set(a.state[p]) == set(b.state[q]) == {"step", "sum"}
        assert torch.equal(p, q) and torch.equal(a.state[p]["sum"], b.state[q]["sum"])
        assert torch.equal(a.state[p]["step"], b.state[q]["step"])


def test_adagrad_sparse_gradients_take_torchs_arithmetic():
    def run(cls):
        emb = torch.nn.Embedding(10, 3, sparse=True)
        with torch.no_grad():
            emb.weight.copy_(torch.arange(30, dtype=torch.float32).reshape(10, 3) / 7)
        opt = cls(emb.parameters(), lr=0.1, lr_decay=0.01)
        for s in range(3):
            opt.zero_grad()
            emb(torch.tensor([1, 4, 4, s])).square().sum().backward()
            assert emb.weight.grad.is_sparse
            opt.step()
        return emb.weight.detach(), opt.state[emb.weight]["sum"]

    (pa, sa), (pb, sb) = run(pdt.optim.Adagrad), run(torch.optim.Adagrad)
    assert torch.equal(pa, pb) and torch.equal(sa, sb)
    with pytest.raises(RuntimeError, match="RMSprop does not support sparse gradients"):
        emb = torch.nn.Embedding(4, 2, sparse=True)
        opt = pdt.optim.RMSprop(emb.parameters())
        emb(torch.tensor([1])).sum().backward()
        opt.step()


def test_adagrad_state_dict_before_the_first_step_matches_torchs():
    """torch's Adagrad creates its state in the constructor: so does ours, and the two state_dicts agree before any step."""
    pa = _cpu_params()
    pb = [p.detach().clone().requires_grad_() for p in pa]
    sa = pdt.optim.Adagrad(pa, lr=0.1, initial_accumulator_value=0.25).state_dict()
    sb = torch.optim.Adagrad(pb, lr=0.1, initial_accumulator_value=0.25).state_dict()
    assert sa["param_groups"] == sb["param_groups"] and set(sa["state"]) == set(sb["state"])
    for i in sa["state"]:
        assert set(sa["state"][i]) == set(sb["state"][i]) == {"step", "sum"}
        for k in ("step", "sum"):
            x, y = sa["state"][i][k], sb["state"][i][k]
            assert x.dtype == y.dtype and x.device == y.device and torch.equal(x, y), k


@pytest.mark.parametrize("ours,theirs,kw", [(pdt.optim.RMSprop, torch.optim.RMSprop, dict(momentum=0.9, centered=True, weight_decay=1e-2)),
                                            (pdt.optim.Adagrad, torch.optim.Adagrad, dict(lr_decay=0.05, weight_decay=1e-2))],
                         ids=["rmsprop", "adagrad"])
@pytest.mark.parametrize("direction", ["torch_to_pdt", "pdt_to_torch"])
def test_state_dict_moves_between_pdt_and_torch(ours, theirs, kw, direction):
    """Three steps with one class, the state_dict into the other (and its learning rate, which differs from the new optimizer's),
    three more steps with both: the same parameters and state as continuing with the first."""
    pa = _cpu_params(seed=3)
    pb = [p.detach().clone().requires_grad_() for p in pa]
    src_cls, dst_cls = (theirs, ours) if direction == "torch_to_pdt" else (ours, theirs)
    src = src_cls(pa, lr=1e-2, **kw)
    gen = torch.Generator().manual_seed(4)
    for _ in range(3):
        for p in pa:
            p.grad = torch.randn(p.shape, generator=gen)
        src.step()
    with torch.no_grad():
        for p, q in zip(pa, pb):
            q.copy_(p)
    dst = dst_cls(pb, lr=5.0)
    dst.load_state_dict(copy.deepcopy(src.state_dict()))
    assert dst.param_groups[0]["lr"] == 1e-2 and all(dst.param_groups[0][k] == v for k, v in kw.items())
    for q in pb:
        assert float(dst.state[q]["step"]) == 3.0 and dst.state[q]["step"].dtype == torch.float32
    for _ in range(3):
        for p, q in zip(pa, pb):
            p.grad = torch.randn(p.shape, generator=gen)
            q.grad = p.grad.clone()
        src.step()
        dst.step()
    for p, q in zip(pa, pb):
        assert float(src.state[p]["step"]) == float(dst.state[q]["step"]) == 6.0
        assert torch.equal(p, q)
        for k in src.state[p]:
            assert torch.equal(src.state[p][k], dst.state[q][k]), k


def _perturbed(v):
    if isinstance(v, bool):
        return not v
    return None if v is None else v / 2 + 0.25


@pytest.mark.parametrize("cls", [pdt.optim.RMSprop, pdt.optim.Adagrad], ids=["rmsprop", "adagrad"])
def test_replay_check_covers_every_key_the_update_reads(cls):
    """A graphed step refuses a replay when one of _FIXED_KEYS changed (one tuple comparison per replay): they must be exactly the
    group keys besides lr that change what _hyper hands the kernels (test_sgd_paths.py's method)."""
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
    group["lr"] = 0.05
    opt.sync_lr()   # lr may change


def test_cli_makes_rmsprop_and_adagrad_with_torchs_defaults_and_refuses_amsgrad():
    from pytorch_distributed_train_b200 import cli

    p = [torch.zeros(1, requires_grad=True)]
    for name, cls, theirs in (("rmsprop", pdt.optim.RMSprop, torch.optim.RMSprop), ("adagrad", pdt.optim.Adagrad, torch.optim.Adagrad)):
        opt = cli.make_optimizer(cli.build_parser().parse_args(["--optimizer", name, "--lr", "1e-3"]), p)
        ref = theirs([torch.zeros(1, requires_grad=True)], lr=1e-3)
        assert type(opt) is cls and opt.defaults == ref.defaults
        opt = cli.make_optimizer(cli.build_parser().parse_args(["--optimizer", name, "--weight-decay", "0.5"]), p)
        assert opt.param_groups[0]["weight_decay"] == 0.5
        for flags, msg in ((["--amsgrad"], "--amsgrad applies to Adam and AdamW only"), (["--momentum", "0.9"], "--momentum applies to SGD only")):
            out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py"), "--optimizer", name] + flags,
                                 capture_output=True, text=True, timeout=60, cwd=ROOT)
            assert out.returncode != 0 and msg in out.stderr, out.stderr[-2000:]


@pytest.mark.parametrize("name,state_key", [("rmsprop", "square_avg"), ("adagrad", "sum")])
def test_train_script_checkpoint_and_resume(tmp_path, name, state_key):
    ck = str(tmp_path / f"{name}.pt")
    base = [sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "2", "--backend", "gloo", "--optimizer", name, "--lr", "1e-3",
            "--steps", "3", "--samples", "600", "--log-interval", "3"]
    a = subprocess.run(base + ["--epochs", "1", "--checkpoint", ck], capture_output=True, text=True, timeout=240, cwd=ROOT)
    assert a.returncode == 0 and os.path.exists(ck), a.stderr[-2000:]
    saved = torch.load(ck, map_location="cpu", weights_only=False)["optimizer"]
    assert all(float(st["step"]) == 3.0 and state_key in st for st in saved["state"].values())
    b = subprocess.run(base + ["--epochs", "2", "--resume", ck], capture_output=True, text=True, timeout=240, cwd=ROOT)
    assert b.returncode == 0, b.stderr[-2000:]
    assert "Resumed from" in b.stdout and "Epoch [2/2], Step [3/3]" in b.stdout and "Epoch [1/2]" not in b.stdout


# =====================================================================================================================
# GPU: the multi-tensor kernels
# =====================================================================================================================
def _dev():
    return torch.device("cuda", 0)


def _shapes(count):
    """count parameters of sizes 1, 3, the ConvNet's, 100003, an empty one and 2²⁰ + 3 (its blocks stride 2²⁰/16384 times)."""
    if count == 1:
        return [(2 ** 20 + 3,)]
    base = [(1,), (3,)] + CONVNET + [(100003,), (0,), (2 ** 20 + 3,)]
    return [base[i % len(base)] for i in range(count)]


KERNEL_CASES = [("rmsprop", c) for c in RMSPROP_CONFIGS] + [("adagrad", c) for c in ADAGRAD_CONFIGS]


@pytest.mark.gpu
@pytest.mark.parametrize("count", [1, 48, 49, 100])
@pytest.mark.parametrize("lr_dev", [False, True], ids=["lr_host", "lr_dev"])
@pytest.mark.parametrize("name,cfg", KERNEL_CASES, ids=[f"{n}-{c}" for n, c in KERNEL_CASES])
def test_multi_kernel_matches_float64(name, cfg, lr_dev, count):
    """Four steps of RMSprop.step() / Adagrad.step() over 1, 48, 49 and 100 tensors (the kernel's table holds 48): each step against
    float64 from the values it started from, one launch per 48 tensors, and the end state against torch's class (foreach=False)
    in fp32."""
    from pytorch_distributed_train_b200 import _C

    ours_cls, theirs_cls = PAIRS[0] if name == "rmsprop" else PAIRS[1]
    kw = (RMSPROP_CONFIGS if name == "rmsprop" else ADAGRAD_CONFIGS)[cfg]
    gen = torch.Generator(device=_dev()).manual_seed(count * 100 + KERNEL_CASES.index((name, cfg)))
    shapes = _shapes(count)
    ours = [torch.randn(s, device=_dev(), generator=gen).requires_grad_() for s in shapes]
    theirs = [p.detach().clone().requires_grad_() for p in ours]
    opt = ours_cls(ours, lr=1e-2, **kw)
    ref = theirs_cls(theirs, lr=1e-2, foreach=False, **kw)
    if lr_dev:
        opt._lr_on_device = True   # what GraphedTrainStep sets: the kernels read lr from a device scalar
    for s in range(4):
        grads = [torch.randn(sh, device=_dev(), generator=gen) * 10 ** (s % 3 - 1) for sh in shapes]
        for p, q, g in zip(ours, theirs, grads):
            p.grad, q.grad = g.clone(), g.clone()
        snap = _snapshot(opt, ours)
        c0 = _C.kernel_launch_count()
        opt.step()
        assert _C.kernel_launch_count() - c0 == math.ceil(count / 48), "one launch per 48 tensors"
        ref.step()
        _expect((s, count), opt, ours, grads, snap)
    if lr_dev:
        assert opt._lr_dev[0][0].item() == _f32(1e-2)
    for p, q in zip(ours, theirs):
        assert opt.state[p]["step"].is_cuda and opt.state[p]["step"].dtype == torch.float32
        assert float(opt.state[p]["step"]) == float(ref.state[q]["step"]) == 4.0
        assert set(opt.state[p]) == set(ref.state[q])
        assert torch.allclose(p, q, atol=1e-6, rtol=1e-5), (p - q).abs().max()
        for k in opt.state[p]:
            if k != "step":
                assert _close(opt.state[p][k], ref.state[q][k]), (k, (opt.state[p][k] - ref.state[q][k]).abs().max())


@pytest.mark.gpu
@pytest.mark.parametrize("ours_cls,theirs_cls,kw", [(pdt.optim.RMSprop, torch.optim.RMSprop, dict(momentum=0.9, centered=True)),
                                                    (pdt.optim.Adagrad, torch.optim.Adagrad, dict(lr_decay=0.1))],
                         ids=["rmsprop", "adagrad"])
def test_nan_gradient_stays_in_its_element_as_in_torch(ours_cls, theirs_cls, kw):
    """A NaN gradient leaves NaN in that element's state and parameter for good, as torch's arithmetic does, and every other element
    is bit for bit what a run without the NaN gives."""
    shapes = [(300,), (17, 5)]
    runs = []
    for poison in (True, False):
        ours = [torch.randn(s, device=_dev(), generator=torch.Generator(device=_dev()).manual_seed(1)).requires_grad_() for s in shapes]
        theirs = [p.detach().clone().requires_grad_() for p in ours]
        a, b = ours_cls(ours, lr=1e-2, **kw), theirs_cls(theirs, lr=1e-2, foreach=False, **kw)
        g = torch.Generator(device=_dev()).manual_seed(2)
        for s in range(5):
            gs = [torch.randn(sh, device=_dev(), generator=g) for sh in shapes]
            if poison and s == 2:
                gs[0][123] = float("nan")
            for p, q, gr in zip(ours, theirs, gs):
                p.grad, q.grad = gr.clone(), gr.clone()
            a.step()
            b.step()
        runs.append((ours, a, theirs, b))
    (ours, a, theirs, b), (clean, ca, _, _) = runs
    assert torch.isnan(ours[0][123])
    for p, q, c in zip(ours, theirs, clean):
        keep = ~torch.isnan(p)
        assert int((~keep).sum()) == (1 if p is ours[0] else 0)
        assert torch.equal(p[keep], c[keep]), "the other elements must be unaffected"
        for x, y in [(p, q)] + [(a.state[p][k], b.state[q][k]) for k in a.state[p] if k != "step"]:
            assert torch.equal(torch.isnan(x), torch.isnan(y))
            assert _close(x, y)
        for k in a.state[p]:
            if k != "step":
                assert torch.equal(a.state[p][k][keep], ca.state[c][k][keep]), k


# =====================================================================================================================
# GPU: the riders of the last backward kernel
# =====================================================================================================================
RIDER_OPTS = {"rmsprop": (pdt.optim.RMSprop, dict(lr=1e-3)),
              "rmsprop_centered_momentum": (pdt.optim.RMSprop, dict(lr=1e-3, momentum=0.9, centered=True, weight_decay=1e-2)),
              "adagrad": (pdt.optim.Adagrad, dict(lr=1e-2, lr_decay=0.1, weight_decay=1e-2, maximize=True))}


@contextlib.contextmanager
def _one_gpu():
    from mp_helpers import free_port

    torch.cuda.set_device(0)
    pdt.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{free_port()}", world_size=1, rank=0)
    try:
        yield
    finally:
        pdt.destroy_process_group()


def _batch(seed, rows=100):
    g = torch.Generator(device=_dev()).manual_seed(seed)
    return torch.rand(rows, 1, 28, 28, device=_dev(), generator=g), torch.randint(0, 10, (rows,), device=_dev(), generator=g)


def _separate_step(opt, params, grads, before):
    """ops.rmsprop_step / ops.adagrad_step of the gradients the rider used, from clones of the state the rider started from: the
    parameters and state it leaves."""
    from pytorch_distributed_train_b200 import ops

    ps = [b[0].clone() for b in before]
    sts = [{k: v.clone() for k, v in b[1].items()} for b in before]
    group = opt.param_groups[0]
    hyper = opt._hyper(0, group, _dev())
    if isinstance(opt, pdt.optim.RMSprop):
        centered = hyper.pop("centered")
        ops.rmsprop_step(ps, grads, [s["square_avg"] for s in sts], [s["step"] for s in sts], **hyper,
                         momentum_buffers=[s["momentum_buffer"] for s in sts] if group["momentum"] > 0 else None,
                         grad_avgs=[s["grad_avg"] for s in sts] if centered else None)
    else:
        ops.adagrad_step(ps, grads, [s["sum"] for s in sts], [s["step"] for s in sts], **hyper)
    return ps, sts


def _assert_same_as_separate(what, opt, params, grads, before):
    ps, sts = _separate_step(opt, params, [g.clone() for g in grads], before)
    for i, (p, q, st) in enumerate(zip(params, ps, sts)):
        assert torch.equal(p.detach(), q), (what, i, "param", (p - q).abs().max().item())
        for k, v in st.items():
            assert torch.equal(opt.state[p][k], v), (what, i, k)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain", "clip2", "clipinf", "accumulate2"])
@pytest.mark.parametrize("name", list(RIDER_OPTS))
def test_rider_matches_float64_of_its_own_gradients(name, mode):
    """The last backward kernel's RMSprop / Adagrad update of all ten ConvNet parameters against float64 of the gradients it stored
    in .grad (clipped, or accumulated over two micro-batches, where it does that first), with the lr in a device scalar; without
    clipping also bit for bit what ops.rmsprop_step / ops.adagrad_step make of those gradients."""
    from pytorch_distributed_train_b200.engine import GraphedTrainStep
    from pytorch_distributed_train_b200.ops import functional as OF

    cls, kw = RIDER_OPTS[name]
    torch.manual_seed(3)
    model = pdt.models.ConvNet(fused=True).to(_dev())
    opt = cls(model.parameters(), **kw)
    opt._lr_on_device = True   # what GraphedTrainStep sets: the kernel reads lr from a device scalar
    crit = pdt.nn.CrossEntropyLoss()

    def before_step():
        params = list(model.parameters())
        for p in params:   # RMSprop creates its state lazily: the first step starts from zeros
            opt._state(p, opt.param_groups[0])
        return params, _snapshot(opt, params), [(p.detach().clone(), {k: v.clone() for k, v in opt.state[p].items()}) for p in params]

    if mode == "accumulate2":
        with _one_gpu():
            x, t = _batch(0, 200)
            step = GraphedTrainStep(pdt.DistributedDataParallel(model, device_ids=[0]), crit, opt, (x, t), warmup=2,
                                    accumulation_steps=2, double_buffer_inputs=False)
            assert step._riding and step.accumulates_in_kernel and step.kernels_per_replay == 6, step.kernels_per_replay
            for s in range(3):
                params, snap, before = before_step()
                x, t = _batch(10 + s, 200)
                step(x, t)
                torch.cuda.synchronize()
                grads = [p.grad for p in params]
                _expect(s, opt, params, grads, snap)
                _assert_same_as_separate(s, opt, params, grads, before)
            opt.stop_riding()
        return
    clip = None
    if mode != "plain":
        norm_out = torch.zeros(1, device=_dev())
        clip = (0.05, 2.0 if mode == "clip2" else math.inf, norm_out)
    assert opt.ride_on_backward(model, clip=clip) and OF._sgd_rider.owner is opt
    try:
        for s in range(3):
            params, snap, before = before_step()
            x, t = _batch(s)
            opt.zero_grad()
            loss = crit(model(x), t)
            with OF.sgd_rider_enabled():
                loss.backward()
            assert opt._rode, "the backward kernel should have applied the update"
            opt.step()
            torch.cuda.synchronize()
            grads = [p.grad for p in params]
            if clip is not None:
                assert norm_out.item() > clip[0], "the gradients must have been clipped"
            _expect(s, opt, params, grads, snap)
            if clip is None:
                _assert_same_as_separate(s, opt, params, grads, before)
    finally:
        opt.stop_riding()


# =====================================================================================================================
# GPU: GraphedTrainStep
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain", "clip", "accumulate"])
@pytest.mark.parametrize("name", ["rmsprop", "adagrad"])
def test_graphed_step_is_three_launches_per_batch_and_follows_torch(name, mode):
    """engine.GraphedTrainStep with pdt.optim.RMSprop / Adagrad on one GPU: the update rides on the last backward kernel, so a replay
    is 3 launches (also with max_grad_norm, 3k with accumulation_steps=k), and 20 replays follow an eager loop with torch's class
    within bench.py's verification tolerance."""
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    ours_cls, theirs_cls = PAIRS[0] if name == "rmsprop" else PAIRS[1]
    lr = 1e-3 if name == "rmsprop" else 1e-2
    k = 2 if mode == "accumulate" else 1
    max_norm = 1.0 if mode == "clip" else None
    with _one_gpu():
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(_dev())
        opt = ours_cls(model.parameters(), lr)
        ddp = pdt.DistributedDataParallel(model, device_ids=[0])
        crit = pdt.nn.CrossEntropyLoss()
        batches = [_batch(90 + i, 100 * k) for i in range(4)]
        step = GraphedTrainStep(ddp, crit, opt, batches[0], warmup=3, max_grad_norm=max_norm, accumulation_steps=k)
        assert step._riding and step.kernels_per_replay == 3 * k, step.kernels_per_replay
        # the reference starts where the engine's eager warm-up steps left the model and the optimizer
        ref = pdt.models.ConvNet().to(_dev())
        ref.load_state_dict(model.state_dict())
        ropt = theirs_cls(ref.parameters(), lr, foreach=False)
        ropt.load_state_dict(copy.deepcopy(opt.state_dict()))   # torch would otherwise share our state tensors
        steps0 = [float(st["step"]) for st in opt.state.values()]
        assert min(steps0) >= 3
        for i in range(20):
            x, t = batches[i % 4]
            step(x, t, inputs_ready=True)
            ropt.zero_grad()
            for j in range(k):
                (crit(ref(x[j * 100:(j + 1) * 100]), t[j * 100:(j + 1) * 100]) / k).backward()
            if max_norm is not None:
                torch.nn.utils.clip_grad_norm_(ref.parameters(), max_norm)
            ropt.step()
        torch.cuda.synchronize()
        assert all(float(st["step"]) == s + 20 for st, s in zip(opt.state.values(), steps0)), "one step per replay"
        keep = [(p, q) for (n, p), q in zip(model.named_parameters(), ref.parameters()) if n not in NOISE]
        err = (_flat([p for p, _ in keep]) - _flat([q for _, q in keep])).abs().max().item() / _flat([q for _, q in keep]).abs().max().item()
        assert err < 2e-2, err


@pytest.mark.gpu
# the replays run the update, never optimizer.step() itself, which torch's schedulers expect to see before their own step
@pytest.mark.filterwarnings("ignore:Detected call of `lr_scheduler.step\\(\\)` before `optimizer.step\\(\\)`")
@pytest.mark.parametrize("name", list(RIDER_OPTS))
def test_graphed_step_follows_a_learning_rate_schedule(name):
    """A LambdaLR that alternates lr between its value and 0, stepped between replays: a replay at lr 0 leaves every parameter
    bitwise unchanged (p − 0·u is p), and a replay at lr > 0 matches float64 of that replay's gradients at the scheduled lr.  For
    Adagrad the decayed rate lr / (1 + s·lr_decay) follows the step count s, which advances on every replay — torch's Adagrad
    computes it on the host, so a captured step of torch's class would replay the captured rate."""
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    cls, kw = RIDER_OPTS[name]
    with _one_gpu():
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(_dev())
        opt = cls(model.parameters(), **kw)
        crit = pdt.nn.CrossEntropyLoss()
        xs = [_batch(20 + i) for i in range(4)]
        step = GraphedTrainStep(pdt.DistributedDataParallel(model, device_ids=[0]), crit, opt, xs[0], warmup=3, double_buffer_inputs=False)
        assert step._riding
        sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda e: 0.0 if e % 3 == 1 else 1.0 / (1 + e))
        for i in range(9):
            lr = opt.param_groups[0]["lr"]
            assert lr == (0.0 if i % 3 == 1 else kw["lr"] * (1.0 / (1 + i)))
            params = list(model.parameters())
            snap = _snapshot(opt, params)
            step(*xs[i % 4], inputs_ready=True)
            torch.cuda.synchronize()
            if lr == 0.0:
                assert torch.equal(_flat(params), snap["p"]), (i, "a replay at lr 0 changed the parameters")
                assert float(opt.state[params[0]]["step"]) == snap["step"] + 1
            else:
                # the oracle decays lr with the step count this replay started from
                _expect(i, opt, params, [p.grad for p in params], snap)
            sched.step()
        opt.stop_riding()
