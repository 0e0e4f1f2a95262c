"""pdt.optim.NAdam and pdt.optim.RAdam: torch's constructors, state and reference arithmetic on the CPU; on the GPU the multi-tensor
kernels (nadam_multi_kernel, radam_multi_kernel) and the riders of the ConvNet's last backward kernel against float64, one step at a
time from the values the step started from, at bounds derived from their roundings (``_nadam64``, ``_radam64``); GraphedTrainStep
with both, across RAdam's switch to the rectified update and under a learning-rate schedule; checkpoint and resume."""
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
# the ConvNet's biases of the two convolutions feed a BatchNorm: their gradient is rounding noise, which Adam-type updates scale up
# to full-size steps, so comparisons of two different gradient paths leave them out (as test_adam.py does)
NOISE = ("layer1.0.bias", "layer2.0.bias")
PAIRS = {"nadam": (pdt.optim.NAdam, torch.optim.NAdam), "radam": (pdt.optim.RAdam, torch.optim.RAdam)}
NADAM_CONFIGS = {"plain": {}, "wd": dict(weight_decay=1e-2), "decoupled": dict(weight_decay=1e-2, decoupled_weight_decay=True),
                 "maximize": dict(maximize=True), "momentum_decay": dict(momentum_decay=0.3)}
# beta2 = 0.75: ρ∞ = 7, so the rectified update starts later (step 8) than with the default (step 6); beta2 = 0.5: ρ∞ = 3, never
RADAM_CONFIGS = {"plain": {}, "wd": dict(weight_decay=1e-2), "decoupled": dict(weight_decay=1e-2, decoupled_weight_decay=True),
                 "maximize": dict(maximize=True), "beta2_late": dict(betas=(0.9, 0.75)), "beta2_never": dict(betas=(0.9, 0.5))}
CONFIGS = {"nadam": NADAM_CONFIGS, "radam": RADAM_CONFIGS}


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def _flat(ts):
    return torch.cat([t.detach().double().reshape(-1) for t in ts]) if ts else torch.zeros(0, dtype=torch.float64)


# =====================================================================================================================
# float64 oracles with their rounding bounds
# =====================================================================================================================
def _nadam_mu(beta1, psi, t):
    return beta1 * (1.0 - 0.5 * 0.96 ** (t * psi))


def _mu_product_next(mp, beta1, psi, step):
    """torch's ``mu_product *= mu`` on its fp32 state tensor, for the step that starts at count ``step``."""
    t = torch.tensor(float(mp), dtype=torch.float32)
    t *= _nadam_mu(beta1, psi, step + 1.0)
    return float(t)


def _rho(beta2, t):
    rho_inf = 2 / (1 - beta2) - 1
    return rho_inf, rho_inf - 2 * t * (beta2 ** t) / (1 - beta2 ** t)


def radam_rectified(beta2, t):
    """Whether torch's RAdam takes the rectified update at step t (ρ_t > 5)."""
    return _rho(beta2, t)[1] > 5.0


def _sqrt_err(x, e):
    """Error bound of sqrt(x) when x carries an error of at most e: e / (2·sqrt(x)) to first order, and never more than sqrt(e)."""
    return torch.minimum(e / (2 * x.clamp_min(1e-300).sqrt()), e.sqrt())


def _moments(g, p, m, v, lr, beta1, beta2, weight_decay, decoupled, maximize):
    """The part NAdam and RAdam share: the gradient g' (weight decay), the parameter p' (decoupled decay) and the moments m', v',
    each with its error bound.  The kernels negate for maximize (exact), then round once in each of: the L2 fma g' = wd·p + g, or
    p' = p·fp32(1 − lr·wd) (the factor rounded, then the product); g' − m and the lerp fma m' = (1 − β1)(g' − m) + m; (1 − β2)·g',
    β2·v and the fma v' = (1 − β2)g'·g' + β2·v.  1 − β1, β2, 1 − β2 and the L2 weight decay are hyper-parameters rounded to fp32."""
    omb1, b2, omb2, wd = _f32(1.0 - beta1), _f32(beta2), _f32(1.0 - beta2), _f32(weight_decay)
    g = -g if maximize else g
    e_g, e_p = torch.zeros_like(g), torch.zeros_like(g)
    if weight_decay and decoupled:
        p = p * (1.0 - lr * weight_decay)
        e_p = 2 * EPS * p.abs()
    elif weight_decay:
        g = g + wd * p
        e_g = EPS * g.abs()
    d = g - m
    m1 = m + omb1 * d
    e_m = EPS * (omb1 * d.abs() + m1.abs()) + omb1 * e_g
    v1 = b2 * v + omb2 * g * g
    e_v = EPS * (2 * omb2 * g * g + b2 * v + v1) + 2 * omb2 * g.abs() * e_g
    return g, e_g, p, e_p, m1, e_m, v1, e_v


def _nadam64(g, p, m, v, step, mu_product, lr, beta1, beta2, eps, weight_decay, momentum_decay, decoupled, maximize):
    """torch.optim.NAdam's step of flat float64 vectors from the values p, m (exp_avg), v (exp_avg_sq), the step count and mu_product
    the kernel started from, with lr as the kernel reads it.  Returns (reference, bound) pairs for p, exp_avg and exp_avg_sq.

    Past _moments the kernels (nadam_multi_kernel, the rider's nadam_apply) round once in each of: the three factors c_g, c_m, bc2
    (formed in double, each rounded to fp32 once); q = v'/bc2; sqrt; + eps; c_m·m'; the fma n = c_g·g' + c_m·m'; the quotient
    u = n/d; p − u.  Π_t, the product torch rounds to fp32, is part of the arithmetic and is formed as torch forms it.  Each rounding
    is ≤ ε = 2⁻²⁴ of its result, the errors of the inputs of each operation are carried through it to first order (through sqrt by
    _sqrt_err, through a division by |δx|/d + |x/d|·δd/(d − δd)), and the bound is twice the first-order sum."""
    eps = _f32(eps)
    t = step + 1.0
    mu, mu_next = _nadam_mu(beta1, momentum_decay, t), _nadam_mu(beta1, momentum_decay, t + 1.0)
    prod = _mu_product_next(mu_product, beta1, momentum_decay, step)
    c_g, c_m, bc2 = lr * (1.0 - mu) / (1.0 - prod), lr * mu_next / (1.0 - prod * mu_next), 1.0 - beta2 ** t
    g, e_g, p, e_p, m1, e_m, v1, e_v = _moments(g, p, m, v, lr, beta1, beta2, weight_decay, decoupled, maximize)
    q = v1 / bc2
    e_q = 2 * EPS * q + e_v / bc2
    root = q.sqrt()
    d = root + eps
    e_d = _sqrt_err(q, e_q) + EPS * root + EPS * d
    n = c_g * g + c_m * m1
    # the fma's rounding, the product c_m·m', the two factors' roundings, and the errors of g' and m'
    e_n = EPS * n.abs() + 2 * EPS * c_m * m1.abs() + EPS * c_g * g.abs() + c_g * e_g + c_m * e_m
    u = n / d
    e_u = EPS * u.abs() + e_n / d + u.abs() * e_d / (d - e_d)
    p1 = p - u
    e_p1 = e_p + EPS * p1.abs() + e_u
    return (p1, 2 * e_p1), (m1, 2 * e_m), (v1, 2 * e_v)


def _radam64(g, p, m, v, step, lr, beta1, beta2, eps, weight_decay, decoupled, maximize):
    """torch.optim.RAdam's step of flat float64 vectors from the values p, m, v and the step count the kernel started from, with lr
    as the kernel reads it.  Returns (reference, bound) pairs for p, exp_avg and exp_avg_sq.

    The branch (ρ_t > 5) is taken from the step count as torch takes it.  Past _moments the kernels (radam_multi_kernel, the
    rider's radam_apply) round once in each of: the step size f (lr·rect·sqrt(bc2)/bc1 or lr/bc1, in double, rounded to fp32 once);
    rectified: sqrt(v'), + eps and the division u = m'/den; the fma p − f·(u or m').  Errors are carried as in _nadam64, and the
    bound is twice the first-order sum."""
    eps = _f32(eps)
    t = step + 1.0
    bc1, bc2 = 1.0 - beta1 ** t, 1.0 - beta2 ** t
    rho_inf, rho_t = _rho(beta2, t)
    g, e_g, p, e_p, m1, e_m, v1, e_v = _moments(g, p, m, v, lr, beta1, beta2, weight_decay, decoupled, maximize)
    if rho_t > 5.0:
        rect = math.sqrt((rho_t - 4) * (rho_t - 2) * rho_inf / ((rho_inf - 4) * (rho_inf - 2) * rho_t))
        f = lr * rect * math.sqrt(bc2) / bc1
        root = v1.sqrt()
        den = root + eps
        e_den = _sqrt_err(v1, e_v) + EPS * root + EPS * den
        u = m1 / den
        e_u = EPS * u.abs() + e_m / den + u.abs() * e_den / (den - e_den)
    else:
        f, u, e_u = lr / bc1, m1, e_m
    p1 = p - f * u
    e_p1 = e_p + EPS * p1.abs() + f * e_u + EPS * f * u.abs()
    return (p1, 2 * e_p1), (m1, 2 * e_m), (v1, 2 * e_v)


def _check(what, got, ref_bound):
    ref, bound = ref_bound
    err = (got.double() - ref).abs()
    ok = err <= bound
    assert bool(ok.all()), (what, int((~ok).sum()), (err - bound).max().item(), (err / bound.clamp_min(1e-300)).max().item())


def _state_of(opt, params, key):
    return _flat([opt.state[p][key] for p in params])


def _snapshot(opt, params):
    """The flat values a NAdam or RAdam step starts from (zeros before the first step), and the first parameter's step count and
    mu_product."""
    snap = {"p": _flat(params)}
    st0 = opt.state[params[0]]
    for key in ("exp_avg", "exp_avg_sq"):
        snap[key] = _state_of(opt, params, key) if key in st0 else torch.zeros_like(snap["p"])
    snap["step"] = float(st0["step"]) if "step" in st0 else 0.0
    snap["mu_product"] = float(st0["mu_product"]) if "mu_product" in st0 else 1.0
    return snap


def _lr_read(opt, group):
    """The learning rate as the kernels read it: fp32 from the device scalar when the optimizer keeps one, else the host's value."""
    return _f32(group["lr"]) if (group.get("capturable") or opt._lr_on_device) else group["lr"]


def _expect(what, opt, params, grads, snap):
    """Every parameter and state tensor of one NAdam or RAdam step against float64 from the snapshot the step started from; step
    (and mu_product) advanced exactly as torch's fp32 state tensors are."""
    g, grp = _flat(grads), opt.param_groups[0]
    beta1, beta2 = grp["betas"]
    common = (g, snap["p"], snap["exp_avg"], snap["exp_avg_sq"], snap["step"])
    if isinstance(opt, pdt.optim.NAdam):
        rp, rm, rv = _nadam64(*common, snap["mu_product"], _lr_read(opt, grp), beta1, beta2, grp["eps"], grp["weight_decay"],
                              grp["momentum_decay"], grp["decoupled_weight_decay"], grp["maximize"])
        want = _mu_product_next(snap["mu_product"], beta1, grp["momentum_decay"], snap["step"])
        assert all(float(opt.state[p]["mu_product"]) == want for p in params), (what, "mu_product")
    else:
        rp, rm, rv = _radam64(*common, _lr_read(opt, grp), beta1, beta2, grp["eps"], grp["weight_decay"], grp["decoupled_weight_decay"],
                              grp["maximize"])
    _check((what, "exp_avg"), _state_of(opt, params, "exp_avg"), rm)
    _check((what, "exp_avg_sq"), _state_of(opt, params, "exp_avg_sq"), rv)
    _check((what, "param"), _flat(params), rp)
    assert all(float(opt.state[p]["step"]) == snap["step"] + 1 for p in params), (what, "step")


# =====================================================================================================================
# CPU
# =====================================================================================================================
def test_radam_configs_switch_where_the_tests_say():
    assert [radam_rectified(0.999, t) for t in range(1, 9)] == [False] * 5 + [True] * 3
    assert [radam_rectified(0.75, t) for t in range(1, 12)] == [False] * 7 + [True] * 4
    assert not any(radam_rectified(0.5, t) for t in range(1, 200))


@pytest.mark.parametrize("name", list(PAIRS))
def test_defaults_match_torch(name):
    ours, theirs = PAIRS[name]
    a, b = ours([torch.zeros(3, requires_grad=True)]), theirs([torch.zeros(3, requires_grad=True)])
    assert a.defaults == b.defaults
    ga, gb = dict(a.param_groups[0]), dict(b.param_groups[0])
    ga.pop("params"), gb.pop("params")
    assert ga == gb


BAD = [dict(lr=-1.0), dict(eps=-1e-8), dict(betas=(1.0, 0.999)), dict(betas=(0.9, -0.1)), dict(weight_decay=-1.0),
       dict(lr=torch.tensor([0.1, 0.2]))]


@pytest.mark.parametrize("name", list(PAIRS))
def test_constructor_errors_match_torch(name):
    ours, theirs = PAIRS[name]
    for kw in BAD + ([dict(momentum_decay=-1e-3)] if name == "nadam" else []):
        with pytest.raises(ValueError) as mine:
            ours([torch.zeros(2, requires_grad=True)], **kw)
        with pytest.raises(ValueError) as ref:
            theirs([torch.zeros(2, requires_grad=True)], **kw)
        assert str(mine.value) == str(ref.value), kw


def _cpu_params(dtype=torch.float32, complex_too=False, seed=0):
    g = torch.Generator().manual_seed(seed)
    ps = [torch.randn(s, generator=g, dtype=dtype).requires_grad_() for s in [(5, 3), (7,), (1,)]]
    if complex_too:
        ps.append(torch.randn(4, generator=g, dtype=torch.complex64).requires_grad_())
    return ps


CPU_CASES = [(n, c) for n in PAIRS for c in CONFIGS[n]]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("name,cfg", CPU_CASES, ids=[f"{n}-{c}" for n, c in CPU_CASES])
def test_reference_step_matches_torch_bit_for_bit(name, cfg, dtype):
    """CPU parameters (and a complex one) take torch's single-tensor arithmetic: ten steps, across RAdam's switch to the rectified
    update, equal torch.optim.NAdam / RAdam(foreach=False) bit for bit, state keys included."""
    ours, theirs = PAIRS[name]
    kw = CONFIGS[name][cfg]
    pa = _cpu_params(dtype, complex_too=True)
    pb = [p.detach().clone().requires_grad_() for p in pa]
    a, b = ours(pa, lr=1e-2, **kw), theirs(pb, lr=1e-2, foreach=False, **kw)
    gen = torch.Generator().manual_seed(1)
    for _ in range(10):
        for p, q in zip(pa, pb):
            p.grad = torch.randn(p.shape, generator=gen, dtype=p.dtype)
            q.grad = p.grad.clone()
        a.step()
        b.step()
    want = {"step", "exp_avg", "exp_avg_sq"} | ({"mu_product"} if name == "nadam" else set())
    for p, q in zip(pa, pb):
        assert set(a.state[p]) == set(b.state[q]) == want
        assert torch.equal(p, q)
        for k in want:
            assert a.state[p][k].dtype == b.state[q][k].dtype and torch.equal(a.state[p][k], b.state[q][k]), k


def test_sparse_gradients_are_refused_as_torch_refuses_them():
    for cls, msg in ((pdt.optim.NAdam, "NAdam does not support sparse gradients"), (pdt.optim.RAdam, "RAdam does not support sparse gradients")):
        emb = torch.nn.Embedding(4, 2, sparse=True)
        opt = cls(emb.parameters())
        emb(torch.tensor([1])).sum().backward()
        with pytest.raises(RuntimeError, match=msg):
            opt.step()


@pytest.mark.parametrize("steps_before", [0, 1, 3], ids=["fresh", "one_step", "three_steps"])
@pytest.mark.parametrize("direction", ["torch_to_pdt", "pdt_to_torch"])
@pytest.mark.parametrize("name", list(PAIRS))
def test_state_dict_moves_between_pdt_and_torch(name, direction, steps_before):
    """0, 1 or 3 steps with one class, the state_dict into the other (and its learning rate, which differs from the new optimizer's),
    three more steps with both: the same parameters and state as continuing with the first."""
    ours, theirs = PAIRS[name]
    kw = dict(weight_decay=1e-2, momentum_decay=5e-3) if name == "nadam" else dict(weight_decay=1e-2, decoupled_weight_decay=True)
    pa = _cpu_params(seed=3)
    pb = [p.detach().clone().requires_grad_() for p in pa]
    src_cls, dst_cls = (theirs, ours) if direction == "torch_to_pdt" else (ours, theirs)
    src = src_cls(pa, lr=1e-2, **kw)
    gen = torch.Generator().manual_seed(4)
    for _ in range(steps_before):
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
        if steps_before:
            assert float(dst.state[q]["step"]) == steps_before and dst.state[q]["step"].dtype == torch.float32
            if name == "nadam":
                assert dst.state[q]["mu_product"].dtype == torch.float32
    for _ in range(3):
        for p, q in zip(pa, pb):
            p.grad = torch.randn(p.shape, generator=gen)
            q.grad = p.grad.clone()
        src.step()
        dst.step()
    for p, q in zip(pa, pb):
        assert float(src.state[p]["step"]) == float(dst.state[q]["step"]) == steps_before + 3
        assert torch.equal(p, q)
        assert set(src.state[p]) == set(dst.state[q])
        for k in src.state[p]:
            assert torch.equal(src.state[p][k], dst.state[q][k]), k


def _perturbed(v):
    if isinstance(v, bool):
        return not v
    if isinstance(v, tuple):
        return tuple(x / 2 + 0.25 for x in v)
    return None if v is None else v / 2 + 0.25


@pytest.mark.parametrize("name", list(PAIRS))
def test_replay_check_covers_every_key_the_update_reads(name):
    """A graphed step refuses a replay when one of _FIXED_KEYS changed: they must be exactly the group keys besides lr that change
    what _hyper hands the kernels (test_sgd_paths.py's method)."""
    cls = PAIRS[name][0]
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


def test_cli_makes_nadam_and_radam_with_torchs_defaults_and_refuses_momentum_and_amsgrad():
    from pytorch_distributed_train_b200 import cli

    p = [torch.zeros(1, requires_grad=True)]
    for name, (cls, theirs) in PAIRS.items():
        opt = cli.make_optimizer(cli.build_parser().parse_args(["--optimizer", name, "--lr", "1e-3"]), p)
        ref = theirs([torch.zeros(1, requires_grad=True)], lr=1e-3)
        assert type(opt) is cls and opt.defaults == ref.defaults
        opt = cli.make_optimizer(cli.build_parser().parse_args(["--optimizer", name, "--weight-decay", "0.5"]), p)
        assert opt.param_groups[0]["weight_decay"] == 0.5 and opt.param_groups[0]["decoupled_weight_decay"] is False
        for flags, msg in ((["--amsgrad"], "--amsgrad applies to Adam and AdamW only"), (["--momentum", "0.9"], "--momentum applies to SGD only")):
            out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py"), "--optimizer", name] + flags,
                                 capture_output=True, text=True, timeout=60, cwd=ROOT)
            assert out.returncode != 0 and msg in out.stderr, out.stderr[-2000:]


@pytest.mark.parametrize("name", list(PAIRS))
def test_train_script_runs_an_epoch_slice_and_resumes(tmp_path, name):
    ck = str(tmp_path / f"{name}.pt")
    base = [sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "2", "--backend", "gloo", "--optimizer", name, "--lr", "1e-3",
            "--steps", "3", "--samples", "600", "--log-interval", "3"]
    a = subprocess.run(base + ["--epochs", "1", "--checkpoint", ck], capture_output=True, text=True, timeout=240, cwd=ROOT)
    assert a.returncode == 0 and os.path.exists(ck), a.stderr[-2000:]
    assert "Epoch [1/1], Step [3/3]" in a.stdout, a.stdout[-2000:]
    saved = torch.load(ck, map_location="cpu", weights_only=False)["optimizer"]
    keys = {"step", "exp_avg", "exp_avg_sq"} | ({"mu_product"} if name == "nadam" else set())
    assert all(float(st["step"]) == 3.0 and set(st) == keys for st in saved["state"].values())
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
    base = [(1,), (3,)] + CONVNET + [(100003,), (0,), (2 ** 20 + 3,)]
    return [base[i % len(base)] for i in range(count)]


KERNEL_CASES = [(n, c) for n in PAIRS for c in CONFIGS[n]]


@pytest.mark.gpu
@pytest.mark.parametrize("lr_dev", [False, True], ids=["lr_host", "lr_dev"])
@pytest.mark.parametrize("name,cfg", KERNEL_CASES, ids=[f"{n}-{c}" for n, c in KERNEL_CASES])
def test_multi_kernel_matches_float64(name, cfg, lr_dev):
    """Eleven steps of NAdam.step() / RAdam.step() over 61 tensors (two launches: the kernel's table holds 48), across RAdam's switch
    to the rectified update: each step against float64 from the values it started from, step and mu_product exactly as torch
    advances its fp32 state, and the end state against torch's class (foreach=False) in fp32."""
    from pytorch_distributed_train_b200 import _C

    ours_cls, theirs_cls = PAIRS[name]
    kw = CONFIGS[name][cfg]
    count = 61
    gen = torch.Generator(device=_dev()).manual_seed(KERNEL_CASES.index((name, cfg)))
    shapes = _shapes(count)
    ours = [torch.randn(s, device=_dev(), generator=gen).requires_grad_() for s in shapes]
    theirs = [p.detach().clone().requires_grad_() for p in ours]
    opt = ours_cls(ours, lr=1e-2, **kw)
    ref = theirs_cls(theirs, lr=1e-2, foreach=False, **kw)
    if lr_dev:
        opt._lr_on_device = True   # what GraphedTrainStep sets: the kernels read lr from a device scalar
    branches = set()
    for s in range(11):
        grads = [torch.randn(sh, device=_dev(), generator=gen) * 10 ** (s % 3 - 1) for sh in shapes]
        for p, q, g in zip(ours, theirs, grads):
            p.grad, q.grad = g.clone(), g.clone()
        snap = _snapshot(opt, ours)
        c0 = _C.kernel_launch_count()
        opt.step()
        assert _C.kernel_launch_count() - c0 == 2, "one launch per 48 tensors"
        ref.step()
        _expect(s, opt, ours, grads, snap)
        branches.add(radam_rectified(opt.param_groups[0]["betas"][1], s + 1))
    if name == "radam":
        assert branches == ({False} if cfg == "beta2_never" else {False, True})
    for p, q in zip(ours, theirs):
        assert opt.state[p]["step"].is_cuda and opt.state[p]["step"].dtype == torch.float32
        assert float(opt.state[p]["step"]) == float(ref.state[q]["step"]) == 11.0
        assert set(opt.state[p]) == set(ref.state[q])
        if name == "nadam":   # torch keeps mu_product on the CPU here: the same fp32 products
            assert opt.state[p]["mu_product"].is_cuda and torch.equal(opt.state[p]["mu_product"].cpu(), ref.state[q]["mu_product"])
        assert torch.allclose(p, q, atol=1e-5, rtol=1e-4), (p - q).abs().max()
        for k in ("exp_avg", "exp_avg_sq"):
            scale = float(ref.state[q][k].abs().max()) if q.numel() else 0.0
            assert torch.allclose(opt.state[p][k], ref.state[q][k], rtol=1e-5, atol=1e-7 + 1e-6 * scale), k


# =====================================================================================================================
# GPU: the riders of the last backward kernel
# =====================================================================================================================
RIDER_OPTS = {"nadam": (pdt.optim.NAdam, dict(lr=2e-3)),
              "nadam_decoupled": (pdt.optim.NAdam, dict(lr=2e-3, weight_decay=1e-2, decoupled_weight_decay=True, momentum_decay=0.1)),
              "radam": (pdt.optim.RAdam, dict(lr=1e-3, weight_decay=1e-2)),
              "radam_late": (pdt.optim.RAdam, dict(lr=1e-3, betas=(0.9, 0.75), maximize=True))}


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


def _assert_same_as_step(what, opt, params, grads, before):
    """ops.nadam_step / ops.radam_step — what step() launches when the update does not ride — of the gradients the rider left in
    .grad, from clones of the state the rider started from: bit for bit the parameters and state the rider left."""
    from pytorch_distributed_train_b200 import ops

    ps = [b[0].clone() for b in before]
    sts = [{k: v.clone() for k, v in b[1].items()} for b in before]
    hyper = opt._hyper(0, opt.param_groups[0], _dev())
    gs = [g.clone() for g in grads]
    if isinstance(opt, pdt.optim.NAdam):
        ops.nadam_step(ps, gs, [s["exp_avg"] for s in sts], [s["exp_avg_sq"] for s in sts], [s["mu_product"] for s in sts],
                       [s["step"] for s in sts], **hyper)
    else:
        ops.radam_step(ps, gs, [s["exp_avg"] for s in sts], [s["exp_avg_sq"] for s in sts], [s["step"] for s in sts], **hyper)
    for i, (p, q, st) in enumerate(zip(params, ps, sts)):
        assert torch.equal(p.detach(), q), (what, i, "param", (p - q).abs().max().item())
        for k, v in st.items():
            assert torch.equal(opt.state[p][k], v), (what, i, k)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain", "clip2", "clipinf", "accumulate2"])
@pytest.mark.parametrize("name", list(RIDER_OPTS))
def test_rider_matches_step_and_float64(name, mode):
    """The last backward kernel's NAdam / RAdam update of all ten ConvNet parameters, with the lr in a device scalar, over seven steps
    (across RAdam's switch): bit for bit what step() makes of the gradients the kernel left in .grad (clipped, or accumulated over
    two micro-batches, where it does that first), and within float64's bounds of them."""
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
        for p in params:   # the state is created lazily: the first step starts from zeros
            opt._state(p)
        return params, _snapshot(opt, params), [(p.detach().clone(), {k: v.clone() for k, v in opt.state[p].items()}) for p in params]

    if mode == "accumulate2":
        with _one_gpu():
            x, t = _batch(0, 200)
            step = GraphedTrainStep(pdt.DistributedDataParallel(model, device_ids=[0]), crit, opt, (x, t), warmup=2,
                                    accumulation_steps=2, double_buffer_inputs=False)
            assert step._riding and step.accumulates_in_kernel and step.kernels_per_replay == 6, step.kernels_per_replay
            for s in range(5):
                params, snap, before = before_step()
                x, t = _batch(10 + s, 200)
                step(x, t)
                torch.cuda.synchronize()
                grads = [p.grad for p in params]
                _expect(s, opt, params, grads, snap)
                _assert_same_as_step(s, opt, params, grads, before)
            opt.stop_riding()
        return
    clip = None
    if mode != "plain":
        norm_out = torch.zeros(1, device=_dev())
        clip = (0.05, 2.0 if mode == "clip2" else math.inf, norm_out)
    assert opt.ride_on_backward(model, clip=clip) and OF._sgd_rider.owner is opt
    try:
        for s in range(7):
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
            _assert_same_as_step(s, opt, params, grads, before)
    finally:
        opt.stop_riding()


# =====================================================================================================================
# GPU: GraphedTrainStep
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain", "clip", "accumulate"])
@pytest.mark.parametrize("name", list(RIDER_OPTS))
def test_graphed_step_is_three_launches_per_batch_and_follows_an_eager_loop(name, mode):
    """engine.GraphedTrainStep with pdt.optim.NAdam / RAdam on one GPU: the update rides on the last backward kernel, so a replay is 3
    launches (also with max_grad_norm, 3k with accumulation_steps=k and the accumulation in the kernels).  Twelve replays, the first
    ones before RAdam's switch to the rectified update and the later ones after it: every replay within float64's bounds of its
    own gradients, and the end state close to an eager loop of the same optimizer class; NAdam's mu_product equal to the eager
    run's bit for bit."""
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    cls, kw = RIDER_OPTS[name]
    k = 2 if mode == "accumulate" else 1
    max_norm = 1.0 if mode == "clip" else None
    with _one_gpu():
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(_dev())
        opt = cls(model.parameters(), **kw)
        ddp = pdt.DistributedDataParallel(model, device_ids=[0])
        crit = pdt.nn.CrossEntropyLoss()
        batches = [_batch(90 + i, 100 * k) for i in range(4)]
        # the reference starts from the same weights and runs the engine's eager warm-up steps itself
        ref = pdt.models.ConvNet().to(_dev())
        ref.load_state_dict(model.state_dict())
        ropt = cls(ref.parameters(), **kw)
        step = GraphedTrainStep(ddp, crit, opt, batches[0], warmup=2, max_grad_norm=max_norm, accumulation_steps=k)
        assert step._riding and step.kernels_per_replay == 3 * k, step.kernels_per_replay
        if k > 1:
            assert step.accumulates_in_kernel
        steps0 = float(opt.state[next(iter(model.parameters()))]["step"])
        ref.load_state_dict(model.state_dict())
        ropt.load_state_dict(copy.deepcopy(opt.state_dict()))
        assert steps0 <= 4
        beta2 = opt.param_groups[0]["betas"][1]
        rectified = set()
        for i in range(12):
            x, t = batches[i % 4]
            params = list(model.parameters())
            snap = _snapshot(opt, params)
            step(x, t, inputs_ready=True)
            torch.cuda.synchronize()
            _expect(i, opt, params, [p.grad for p in params], snap)
            rectified.add(radam_rectified(beta2, snap["step"] + 1))
            ropt.zero_grad()
            for j in range(k):
                (crit(ref(x[j * 100:(j + 1) * 100]), t[j * 100:(j + 1) * 100]) / k).backward()
            if max_norm is not None:
                torch.nn.utils.clip_grad_norm_(ref.parameters(), max_norm)
            ropt.step()
        torch.cuda.synchronize()
        if cls is pdt.optim.RAdam:
            assert rectified == {False, True}, "the replays must cross into the rectified update"
        for p, q in zip(model.parameters(), ref.parameters()):
            assert float(opt.state[p]["step"]) == float(ropt.state[q]["step"]) == steps0 + 12, "one step per replay"
            if cls is pdt.optim.NAdam:
                assert torch.equal(opt.state[p]["mu_product"], ropt.state[q]["mu_product"])
        keep = [(p, q) for (n, p), q in zip(model.named_parameters(), ref.parameters()) if n not in NOISE]
        err = (_flat([p for p, _ in keep]) - _flat([q for _, q in keep])).abs().max().item() / _flat([q for _, q in keep]).abs().max().item()
        assert err < 2e-2, err
        opt.stop_riding()


@pytest.mark.gpu
# the replays run the update, never optimizer.step() itself, which torch's schedulers expect to see before their own step
@pytest.mark.filterwarnings("ignore:Detected call of `lr_scheduler.step\\(\\)` before `optimizer.step\\(\\)`")
@pytest.mark.parametrize("name", list(RIDER_OPTS))
def test_graphed_step_follows_a_learning_rate_schedule_and_refuses_new_betas(name):
    """A LambdaLR that alternates lr between a decaying value and 0, stepped between ten replays: a replay at lr 0 leaves every
    parameter bitwise unchanged and still advances the step (and mu_product), and a replay at lr > 0 matches float64 of that replay's
    gradients at the scheduled lr.  Changing betas after the capture is refused by the next replay."""
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    cls, kw = RIDER_OPTS[name]
    with _one_gpu():
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(_dev())
        opt = cls(model.parameters(), **kw)
        crit = pdt.nn.CrossEntropyLoss()
        xs = [_batch(20 + i) for i in range(4)]
        step = GraphedTrainStep(pdt.DistributedDataParallel(model, device_ids=[0]), crit, opt, xs[0], warmup=3, double_buffer_inputs=False)
        assert step._riding and step.kernels_per_replay == 3
        sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda e: 0.0 if e % 3 == 1 else 1.0 / (1 + e))
        for i in range(10):
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
                _expect(i, opt, params, [p.grad for p in params], snap)
            sched.step()
        beta1, beta2 = opt.param_groups[0]["betas"]
        opt.param_groups[0]["betas"] = (beta1 / 2, beta2)
        with pytest.raises(RuntimeError, match="'betas' of param_groups\\[0\\]"):
            step(*xs[0], inputs_ready=True)
        opt.stop_riding()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(RIDER_OPTS))
def test_checkpoint_resume_gives_the_uninterrupted_next_step(tmp_path, name):
    """Four steps, save_checkpoint, one more step; a fresh model and optimizer loaded from the checkpoint take the same fifth step
    bit for bit (step and mu_product come back to the device as fp32)."""
    from pytorch_distributed_train_b200.utils import load_checkpoint, save_checkpoint

    cls, kw = RIDER_OPTS[name]
    crit = pdt.nn.CrossEntropyLoss()

    def make():
        torch.manual_seed(0)
        m = pdt.models.ConvNet().to(_dev())
        return m, cls(m.parameters(), **kw)

    def one_step(m, o, s):
        o.zero_grad()
        crit(m(_batch(s)[0]), _batch(s)[1]).backward()
        o.step()

    model, opt = make()
    for s in range(4):
        one_step(model, opt, s)
    ck = str(tmp_path / "ck.pt")
    save_checkpoint(ck, model, opt, epoch=1)
    one_step(model, opt, 4)
    model2, opt2 = make()
    load_checkpoint(ck, model2, opt2)
    for p in model2.parameters():
        for key in ("step", "mu_product"):
            if key in opt2.state[p]:
                assert opt2.state[p][key].is_cuda and opt2.state[p][key].dtype == torch.float32
    one_step(model2, opt2, 4)
    torch.cuda.synchronize()
    for p, q in zip(model.parameters(), model2.parameters()):
        assert torch.equal(p, q)
        for k in opt.state[p]:
            assert torch.equal(opt.state[p][k], opt2.state[q][k]), k
