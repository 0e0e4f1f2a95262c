"""pdt.optim.Adamax, Adadelta, ASGD and Rprop: torch's constructors, state and reference arithmetic on the CPU; on the GPU the
multi-tensor kernels (adamax_multi_kernel, adadelta_multi_kernel, asgd_multi_kernel, rprop_multi_kernel) and the riders of the
ConvNet's last backward kernel against float64, one step at a time from the values the step started from, at bounds derived from
their roundings (``_adamax64``, ``_adadelta64``, ``_asgd64``, ``_rprop64``); Rprop also bit for bit against torch's single-tensor
Rprop; GraphedTrainStep with all four, under a learning-rate schedule; checkpoint and resume."""
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
# the ConvNet's biases of the two convolutions feed a BatchNorm: their gradient is rounding noise, which sign- and ratio-based
# updates scale up to full-size steps, so comparisons of two different gradient paths leave them out (as test_adam.py does)
NOISE = ("layer1.0.bias", "layer2.0.bias")
PAIRS = {"adamax": (pdt.optim.Adamax, torch.optim.Adamax), "adadelta": (pdt.optim.Adadelta, torch.optim.Adadelta),
         "asgd": (pdt.optim.ASGD, torch.optim.ASGD), "rprop": (pdt.optim.Rprop, torch.optim.Rprop)}
KEYS = {"adamax": ("exp_avg", "exp_inf"), "adadelta": ("square_avg", "acc_delta"), "asgd": ("ax",), "rprop": ("prev", "step_size")}
SCALARS = {"adamax": ("step",), "adadelta": ("step",), "asgd": ("step", "eta", "mu"), "rprop": ("step",)}
# ASGD's t0 = 3: mu stays 1 (ax = p) for the first four steps, then 1 / (t − 3) (the averaging branch)
CONFIGS = {
    "adamax": {"plain": {}, "wd": dict(weight_decay=1e-2), "maximize": dict(maximize=True), "betas": dict(betas=(0.5, 0.9))},
    "adadelta": {"plain": {}, "wd": dict(weight_decay=1e-2), "maximize": dict(maximize=True), "rho": dict(rho=0.5, eps=1e-4)},
    "asgd": {"plain": dict(t0=3), "wd": dict(t0=3, weight_decay=1e-2), "maximize": dict(t0=3, maximize=True),
             "lambd": dict(t0=3, lambd=0.5, alpha=0.5)},
    "rprop": {"plain": {}, "maximize": dict(maximize=True), "etas": dict(etas=(0.3, 1.5)), "bounds": dict(step_sizes=(2e-3, 2e-2))},
}


def _name(opt):
    return next(n for n, (cls, _) in PAIRS.items() if isinstance(opt, cls))


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


def _decayed(g, p, weight_decay, maximize):
    """g' = ±g + wd·p (the kernels negate exactly, then round the fma once) and its error bound."""
    g = -g if maximize else g
    if weight_decay:
        g = g + _f32(weight_decay) * p
        return g, EPS * g.abs()
    return g, torch.zeros_like(g)


def _adamax64(g, p, m, u, step, lr, beta1, beta2, eps, weight_decay, maximize):
    """torch.optim.Adamax's step of flat float64 vectors from the values p, m (exp_avg), u (exp_inf) and the step count the kernel
    started from, with lr as the kernel reads it.  Returns (reference, bound) pairs for p, exp_avg and exp_inf.

    The kernels (adamax_update) round once in each of: g' − m and the lerp fma m' = (1 − β1)(g' − m) + m; β2·u; |g'| + eps; the step
    size clr = lr / (1 − β1^t) (double, rounded to fp32 once); the quotient m'/u'; the fma p − clr·(m'/u').  The maximum carries the
    larger of its inputs' errors; a NaN in either input stays.  Errors of each operation's inputs are carried through it to first
    order, and the bound is twice the first-order sum."""
    omb1, b2, eps = _f32(1.0 - beta1), _f32(beta2), _f32(eps)
    g, e_g = _decayed(g, p, weight_decay, maximize)
    d = g - m
    m1 = m + omb1 * d
    e_m = EPS * (omb1 * d.abs() + m1.abs()) + omb1 * e_g
    a, c = b2 * u, g.abs() + eps
    u1 = torch.where(a.isnan() | (a > c), a, c)
    e_u = torch.maximum(EPS * a.abs(), EPS * c + e_g)
    clr = lr / (1.0 - beta1 ** (step + 1.0))
    q = m1 / u1
    e_q = EPS * q.abs() + e_m / u1 + q.abs() * e_u / (u1 - e_u)
    p1 = p - clr * q
    e_p1 = EPS * p1.abs() + clr * e_q + EPS * clr * q.abs()
    return (p1, 2 * e_p1), (m1, 2 * e_m), (u1, 2 * e_u)


def _adadelta64(g, p, sq, acc, lr, rho, eps, weight_decay, maximize):
    """torch.optim.Adadelta's step of flat float64 vectors from the values p, sq (square_avg) and acc (acc_delta) the kernel started
    from; lr is fp32 (the kernels take it so).  Returns (reference, bound) pairs for p, square_avg and acc_delta.

    The kernels (adadelta_update) round once in each of: (1 − ρ)·g', ρ·sq and the fma sq'; acc + eps, sqrt; sq' + eps, sqrt; the
    quotient r; δ = r·g'; (1 − ρ)·δ, ρ·acc and the fma acc'; the fma p − lr·δ.  Errors are carried as in _adamax64."""
    r32, omr, eps = _f32(rho), _f32(1.0 - rho), _f32(eps)
    g, e_g = _decayed(g, p, weight_decay, maximize)
    s1 = r32 * sq + omr * g * g
    e_s = EPS * (2 * omr * g * g + r32 * sq + s1) + 2 * omr * g.abs() * e_g
    a_ = acc + eps
    ra = a_.sqrt()
    e_ra = _sqrt_err(a_, EPS * a_) + EPS * ra
    s_ = s1 + eps
    rs = s_.sqrt()
    e_rs = _sqrt_err(s_, e_s + EPS * s_) + EPS * rs
    r = ra / rs
    e_r = EPS * r + e_ra / rs + r * e_rs / (rs - e_rs)
    d = r * g
    e_d = EPS * d.abs() + r * e_g + e_r * g.abs()
    acc1 = r32 * acc + omr * d * d
    e_acc = EPS * (2 * omr * d * d + r32 * acc + acc1) + 2 * omr * d.abs() * e_d
    p1 = p - lr * d
    e_p1 = EPS * p1.abs() + lr * e_d
    return (p1, 2 * e_p1), (s1, 2 * e_s), (acc1, 2 * e_acc)


def asgd_schedules(lr, lambd, alpha, t0, t):
    """torch's non-capturable ASGD: the eta and mu it stores after the step that leaves the count at t, rounded to fp32."""
    return _f32(lr / ((1 + lambd * lr * t) ** alpha)), _f32(1 / max(1, t - t0))


def _asgd64(g, p, ax, eta, mu, lambd, weight_decay, maximize):
    """torch.optim.ASGD's step of flat float64 vectors from the values p, ax and the fp32 eta, mu the kernel started from.  Returns
    (reference, bound) pairs for p and ax.

    The kernels (asgd_update) round once in each of: the decay factor fp32(1 − λ·η) (formed as torch forms it: exact here); p·decay;
    the fma p − η·g'; then, where mu != 1, p − ax, its product with mu and the sum ax + (p − ax)·mu (where mu == 1, ax = p)."""
    decay = _f32(1.0 - lambd * eta)
    g, e_g = _decayed(g, p, weight_decay, maximize)
    pd = p * decay
    p1 = pd - eta * g
    e_p1 = EPS * pd.abs() + EPS * p1.abs() + eta * e_g
    if mu == 1.0:
        return (p1, 2 * e_p1), (p1, 2 * e_p1)
    d = p1 - ax
    e_d = e_p1 + EPS * d.abs()
    t = d * mu
    e_t = EPS * t.abs() + mu * e_d
    ax1 = ax + t
    e_ax = EPS * ax1.abs() + e_t
    return (p1, 2 * e_p1), (ax1, 2 * e_ax)


def _rprop64(g, p, prev, ss, etaminus, etaplus, step_min, step_max, maximize):
    """torch.optim.Rprop's step of flat float64 vectors from the values p, prev and step_size the kernel started from.  Returns
    (reference, bound) pairs for p, prev and step_size.

    The sign of the gradient's product with prev is that of the fp32 product (it underflows where torch's does), and the factors are
    fp32(η±), as torch's tensor holds them.  Every operation is exact except the products step_size·f and the difference
    p − sign·step_size, which round once each."""
    g = -g if maximize else g
    prod = (g.float() * prev.float()).double()
    em, ep = _f32(etaminus), _f32(etaplus)
    f = torch.where(prod > 0, ep, torch.where(prod < 0, em, 1.0)).double()
    s1 = (ss * f).clamp(_f32(step_min), _f32(step_max))
    e_s = EPS * s1
    gg = torch.where(f == em, torch.zeros_like(g), g)
    sign = torch.where(gg > 0, 1.0, torch.where(gg < 0, -1.0, 0.0)).double()
    p1 = p - sign * s1
    e_p1 = EPS * p1.abs() + e_s
    return (p1, 2 * e_p1), (gg, torch.zeros_like(gg)), (s1, 2 * e_s)


def _check(what, got, ref_bound):
    ref, bound = ref_bound
    got = got.double()
    nan = ref.isnan()
    assert torch.equal(got.isnan(), nan), (what, "NaN positions differ", int((got.isnan() != nan).sum()))
    err = (got - ref).abs()[~nan]
    ok = err <= bound[~nan]
    assert bool(ok.all()), (what, int((~ok).sum()), (err - bound[~nan]).max().item())


def _bits_equal(a, b):
    """Bit for bit (the sign of a zero included) where not NaN, and NaN in the same places (a NaN's sign and payload carry nothing:
    the GPU's arithmetic returns its canonical NaN where torch's negation flips the sign bit)."""
    nan = a.isnan()
    if a.dtype != b.dtype or not torch.equal(nan, b.isnan()):
        return False
    return torch.equal(a[~nan].view(torch.int32), b[~nan].view(torch.int32))


def _state_of(opt, params, key):
    return _flat([opt.state[p][key] for p in params])


def _snapshot(opt, params):
    """The flat values a step starts from (torch's initial state before the first step), and the first parameter's scalars."""
    name, grp = _name(opt), opt.param_groups[0]
    snap = {"p": _flat(params)}
    st0 = opt.state[params[0]]
    for key in KEYS[name]:
        init = torch.full_like(snap["p"], _f32(grp["lr"])) if key == "step_size" else torch.zeros_like(snap["p"])
        snap[key] = _state_of(opt, params, key) if key in st0 else init
    snap["step"] = float(st0["step"]) if "step" in st0 else 0.0
    snap["eta"] = float(st0["eta"]) if "eta" in st0 else _f32(grp["lr"])
    snap["mu"] = float(st0["mu"]) if "mu" in st0 else 1.0
    return snap


def _lr_read(opt, group):
    """The learning rate as the kernels read it: fp32 from the device scalar when the optimizer keeps one, else the host's value;
    Adadelta's kernels take it in fp32 always."""
    if group.get("capturable") or opt._lr_on_device or isinstance(opt, pdt.optim.Adadelta):
        return _f32(group["lr"])
    return group["lr"]


def _expect(what, opt, params, grads, snap):
    """Every parameter and state tensor of one step against float64 from the snapshot the step started from; step (and ASGD's eta
    and mu) advanced as torch advances its fp32 state."""
    name, g, grp = _name(opt), _flat(grads), opt.param_groups[0]
    p = snap["p"]
    if name == "adamax":
        beta1, beta2 = grp["betas"]
        refs = _adamax64(g, p, snap["exp_avg"], snap["exp_inf"], snap["step"], _lr_read(opt, grp), beta1, beta2, grp["eps"],
                         grp["weight_decay"], grp["maximize"])
    elif name == "adadelta":
        refs = _adadelta64(g, p, snap["square_avg"], snap["acc_delta"], _lr_read(opt, grp), grp["rho"], grp["eps"], grp["weight_decay"],
                           grp["maximize"])
    elif name == "asgd":
        refs = _asgd64(g, p, snap["ax"], snap["eta"], snap["mu"], grp["lambd"], grp["weight_decay"], grp["maximize"])
        eta, mu = asgd_schedules(_lr_read(opt, grp), grp["lambd"], grp["alpha"], grp["t0"], snap["step"] + 1)
        for q in params:
            # the device's pow may differ from the host's in the last bit of the double, which can move the fp32 rounding by one ulp
            assert abs(float(opt.state[q]["eta"]) - eta) <= 2.0 ** -23 * eta, (what, "eta", float(opt.state[q]["eta"]), eta)
            assert float(opt.state[q]["mu"]) == mu, (what, "mu", float(opt.state[q]["mu"]), mu)
    else:
        etaminus, etaplus = grp["etas"]
        step_min, step_max = grp["step_sizes"]
        refs = _rprop64(g, p, snap["prev"], snap["step_size"], etaminus, etaplus, step_min, step_max, grp["maximize"])
    _check((what, "param"), _flat(params), refs[0])
    for key, ref in zip(KEYS[name], refs[1:]):
        _check((what, key), _state_of(opt, params, key), ref)
    assert all(float(opt.state[q]["step"]) == snap["step"] + 1 for q in params), (what, "step")


# =====================================================================================================================
# CPU
# =====================================================================================================================
def test_asgd_config_runs_both_averaging_branches():
    """t0 = 3: mu is 1 after steps 1 … 4 (ax = p at steps 1 … 5), then 1 / (t − 3)."""
    mus = [asgd_schedules(1e-2, 1e-4, 0.75, 3, t)[1] for t in range(1, 12)]
    assert mus[:4] == [1.0] * 4 and all(m < 1.0 for m in mus[4:])


@pytest.mark.parametrize("name", list(PAIRS))
def test_defaults_match_torch(name):
    ours, theirs = PAIRS[name]
    a, b = ours([torch.zeros(3, requires_grad=True)]), theirs([torch.zeros(3, requires_grad=True)])
    assert a.defaults == b.defaults
    ga, gb = dict(a.param_groups[0]), dict(b.param_groups[0])
    ga.pop("params"), gb.pop("params")
    assert ga == gb


BAD = {"adamax": [dict(lr=-1.0), dict(eps=-1e-8), dict(betas=(1.0, 0.999)), dict(betas=(0.9, -0.1)), dict(weight_decay=-1.0)],
       "adadelta": [dict(lr=-1.0), dict(rho=1.5), dict(rho=-0.1), dict(eps=-1e-6), dict(weight_decay=-1.0)],
       "asgd": [dict(lr=-1.0), dict(weight_decay=-1.0)],
       "rprop": [dict(lr=-1.0), dict(etas=(1.2, 0.5)), dict(etas=(0.0, 1.2)), dict(etas=(0.5, 1.0))]}


@pytest.mark.parametrize("name", list(PAIRS))
def test_constructor_errors_match_torch(name):
    ours, theirs = PAIRS[name]
    for kw in BAD[name] + [dict(lr=torch.tensor([0.1, 0.2]))]:
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


CASES = [(n, c) for n in PAIRS for c in CONFIGS[n]]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("name,cfg", CASES, ids=[f"{n}-{c}" for n, c in CASES])
def test_reference_step_matches_torch_bit_for_bit(name, cfg, dtype):
    """CPU parameters (and a complex one) take torch's single-tensor arithmetic: ten steps equal torch's class (foreach=False) bit
    for bit, state keys and dtypes included."""
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
    want = set(KEYS[name]) | set(SCALARS[name])
    for p, q in zip(pa, pb):
        assert set(a.state[p]) == set(b.state[q]) == want
        assert torch.equal(p, q)
        for k in want:
            assert a.state[p][k].dtype == b.state[q][k].dtype and torch.equal(a.state[p][k], b.state[q][k]), k


@pytest.mark.parametrize("name", list(PAIRS))
def test_sparse_gradients_are_refused_as_torch_refuses_them(name):
    for cls in PAIRS[name]:
        emb = torch.nn.Embedding(4, 2, sparse=True)
        opt = cls(emb.parameters())
        emb(torch.tensor([1])).sum().backward()
        with pytest.raises(RuntimeError, match=f"{cls.__name__} does not support sparse gradients"):
            opt.step()


STATE_DICT_KW = {"adamax": dict(weight_decay=1e-2, betas=(0.8, 0.99)), "adadelta": dict(weight_decay=1e-2, rho=0.8),
                 "asgd": dict(weight_decay=1e-2, t0=1), "rprop": dict(etas=(0.4, 1.3))}


@pytest.mark.parametrize("steps_before", [0, 1, 3], ids=["fresh", "one_step", "three_steps"])
@pytest.mark.parametrize("direction", ["torch_to_pdt", "pdt_to_torch"])
@pytest.mark.parametrize("name", list(PAIRS))
def test_state_dict_moves_between_pdt_and_torch(name, direction, steps_before):
    """0, 1 or 3 steps with one class, the state_dict into the other (and its learning rate, which differs from the new optimizer's),
    three more steps with both: the same parameters and state as continuing with the first."""
    ours, theirs = PAIRS[name]
    kw = STATE_DICT_KW[name]
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
            for key in SCALARS[name]:
                assert dst.state[q][key].dtype == torch.float32, key
            assert float(dst.state[q]["step"]) == steps_before
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
    what _hyper hands the kernels (test_sgd_paths.py's method).  lr may change; for Rprop it is not handed to the kernels at all."""
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
    assert "lr" not in cls._FIXED_KEYS
    if name == "rprop":
        assert "lr" not in base
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


def test_cli_makes_the_four_optimizers_with_torchs_defaults_and_refuses_rprop_weight_decay():
    from pytorch_distributed_train_b200 import cli

    p = [torch.zeros(1, requires_grad=True)]
    for name, (cls, theirs) in PAIRS.items():
        opt = cli.make_optimizer(cli.build_parser().parse_args(["--optimizer", name, "--lr", "1e-3"]), p)
        ref = theirs([torch.zeros(1, requires_grad=True)], lr=1e-3)
        assert type(opt) is cls and opt.defaults == ref.defaults
        if name != "rprop":
            opt = cli.make_optimizer(cli.build_parser().parse_args(["--optimizer", name, "--weight-decay", "0.5"]), p)
            assert opt.param_groups[0]["weight_decay"] == 0.5
    for name, flags, msg in (("rprop", ["--weight-decay", "0.1"], "--weight-decay does not apply to Rprop"),
                             ("adadelta", ["--momentum", "0.9"], "--momentum applies to SGD only"),
                             ("asgd", ["--amsgrad"], "--amsgrad applies to Adam and AdamW only")):
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
    keys = set(KEYS[name]) | set(SCALARS[name])
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


def _offset(params, i):
    """Where parameter i starts in the flat vectors of _flat."""
    return sum(p.numel() for p in params[:i])


def _edge_cases(name, s, grads, ours, theirs, opt, ref):
    """The inputs the issue's edge cases need, written identically into both optimizers' gradients and state.  Tensor 2 (400
    elements) takes them.  Adamax: a NaN gradient entry at step 3 (exp_inf keeps it).  Rprop at step 4: prev·g exactly zero, a
    product that underflows in fp32, and a NaN gradient."""
    if name == "adamax" and s == 3:
        grads[2].view(-1)[7] = float("nan")
    if name == "rprop" and s == 4:
        g = grads[2].view(-1)
        for pp, o in ((ours[2], opt), (theirs[2], ref)):
            prev = o.state[pp]["prev"].view(-1)
            prev[0], prev[1], prev[2] = 1.0, 1e-20, 1.0
        g[0], g[1], g[2] = 0.0, 1e-30, float("nan")


@pytest.mark.gpu
@pytest.mark.parametrize("lr_dev", [False, True], ids=["lr_host", "lr_dev"])
@pytest.mark.parametrize("name,cfg", CASES, ids=[f"{n}-{c}" for n, c in CASES])
def test_multi_kernel_matches_float64(name, cfg, lr_dev):
    """Eleven steps of step() over 61 tensors (two launches: the kernel's table holds 48), with the edge cases of _edge_cases: each
    step against float64 from the values it started from, step (and ASGD's eta and mu) as torch advances its fp32 state, and the end
    state close to torch's class (foreach=False); Rprop bit for bit against torch's single-tensor Rprop on the same device at every
    step."""
    from pytorch_distributed_train_b200 import _C

    ours_cls, theirs_cls = PAIRS[name]
    kw = CONFIGS[name][cfg]
    count = 61
    gen = torch.Generator(device=_dev()).manual_seed(CASES.index((name, cfg)))
    shapes = _shapes(count)
    ours = [torch.randn(s, device=_dev(), generator=gen).requires_grad_() for s in shapes]
    theirs = [p.detach().clone().requires_grad_() for p in ours]
    opt = ours_cls(ours, lr=1e-2, **kw)
    ref = theirs_cls(theirs, lr=1e-2, foreach=False, **kw)
    if lr_dev:
        opt._lr_on_device = True   # what GraphedTrainStep sets: the kernels read lr from a device scalar
    mus, clamped = set(), set()
    for s in range(11):
        grads = [torch.randn(sh, device=_dev(), generator=gen) * 10 ** (s % 3 - 1) for sh in shapes]
        if s > 0:
            _edge_cases(name, s, grads, ours, theirs, opt, ref)
        for p, q, g in zip(ours, theirs, grads):
            p.grad, q.grad = g.clone(), g.clone()
        snap = _snapshot(opt, ours)
        mus.add(snap["mu"] == 1.0)
        c0 = _C.kernel_launch_count()
        opt.step()
        assert _C.kernel_launch_count() - c0 == 2, "one launch per 48 tensors"
        ref.step()
        _expect(s, opt, ours, grads, snap)
        if name == "rprop":
            for i, (p, q) in enumerate(zip(ours, theirs)):
                assert _bits_equal(p.detach(), q.detach()), (s, i, "param")
                for k in ("prev", "step_size"):
                    assert _bits_equal(opt.state[p][k], ref.state[q][k]), (s, i, k)
            if s == 4:   # the zero, underflowed and NaN products count as 0: factor 1, and g'' = g
                prev, ss = opt.state[ours[2]]["prev"].view(-1), opt.state[ours[2]]["step_size"].view(-1)
                assert prev[0] == 0.0 and abs(float(prev[1])) == _f32(1e-30) and prev[2].isnan()
                off = _offset(ours, 2)
                assert torch.equal(ss[:3].double(), snap["step_size"][off:off + 3])
            ss = _state_of(opt, ours, "step_size")
            lo, hi = (_f32(v) for v in opt.param_groups[0]["step_sizes"])
            clamped |= {"min"} if bool((ss == lo).any()) else set()
            clamped |= {"max"} if bool((ss == hi).any()) else set()
    if name == "asgd":
        assert mus == {True, False}, "both averaging branches"
    if name == "rprop" and cfg == "bounds":
        assert clamped == {"min", "max"}, clamped
    if name == "adamax":
        assert opt.state[ours[2]]["exp_inf"].view(-1)[7].isnan(), "exp_inf keeps the NaN"
    for p, q in zip(ours, theirs):
        assert opt.state[p]["step"].is_cuda and opt.state[p]["step"].dtype == torch.float32
        assert float(opt.state[p]["step"]) == float(ref.state[q]["step"]) == 11.0
        assert set(opt.state[p]) == set(ref.state[q])
        assert torch.allclose(p, q, atol=1e-5, rtol=1e-4, equal_nan=True), (p - q).abs().max()
        for k in KEYS[name]:
            scale = float(ref.state[q][k].nan_to_num().abs().max()) if q.numel() else 0.0
            assert torch.allclose(opt.state[p][k], ref.state[q][k], rtol=1e-5, atol=1e-7 + 1e-6 * scale, equal_nan=True), k


# =====================================================================================================================
# GPU: the riders of the last backward kernel
# =====================================================================================================================
RIDER_OPTS = {"adamax": (pdt.optim.Adamax, dict(lr=2e-3, weight_decay=1e-2)),
              "adadelta": (pdt.optim.Adadelta, dict(lr=1.0)),
              "asgd": (pdt.optim.ASGD, dict(lr=1e-2, t0=2, lambd=1e-2, weight_decay=1e-3)),
              "rprop": (pdt.optim.Rprop, dict(lr=1e-3, maximize=False))}


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
    """The ops.*_step that step() launches when the update does not ride, of the gradients the rider left in .grad, from clones of
    the state the rider started from: bit for bit the parameters and state the rider left."""
    from pytorch_distributed_train_b200 import ops

    name = _name(opt)
    ps = [b[0].clone() for b in before]
    sts = [{k: v.clone() for k, v in b[1].items()} for b in before]
    hyper = opt._hyper(0, opt.param_groups[0], _dev())
    gs = [g.clone() for g in grads]
    lists = {k: [s[k] for s in sts] for k in sts[0]}
    if name == "adamax":
        ops.adamax_step(ps, gs, lists["exp_avg"], lists["exp_inf"], lists["step"], **hyper)
    elif name == "adadelta":
        ops.adadelta_step(ps, gs, lists["square_avg"], lists["acc_delta"], lists["step"], **hyper)
    elif name == "asgd":
        ops.asgd_step(ps, gs, lists["ax"], lists["step"], lists["eta"], lists["mu"], **hyper)
    else:
        ops.rprop_step(ps, gs, lists["prev"], lists["step_size"], lists["step"], **hyper)
    for i, (p, q, st) in enumerate(zip(params, ps, sts)):
        assert torch.equal(p.detach(), q), (what, i, "param", (p - q).abs().max().item())
        for k, v in st.items():
            assert torch.equal(opt.state[p][k], v), (what, i, k)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain", "clip2", "clipinf", "accumulate2"])
@pytest.mark.parametrize("name", list(RIDER_OPTS))
def test_rider_matches_step_and_float64(name, mode):
    """The last backward kernel's update of all ten ConvNet parameters, with the lr in a device scalar, over seven steps (ASGD across
    its switch to averaging): bit for bit what step() makes of the gradients the kernel left in .grad (clipped, or accumulated over
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
        snap = _snapshot(opt, params)   # before the lazy state exists: torch's initial values
        for p in params:
            opt._state(p, opt.param_groups[0])
        return params, snap, [(p.detach().clone(), {k: v.clone() for k, v in opt.state[p].items()}) for p in params]

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
    """engine.GraphedTrainStep on one GPU: the update rides on the last backward kernel, so a replay is 3 launches (also with
    max_grad_norm, 3k with accumulation_steps=k and the accumulation in the kernels).  Twelve replays: every replay within float64's
    bounds of its own gradients, and the end state close to an eager loop of the same optimizer class.  Rprop's sign-based steps
    turn a gradient's rounding noise into a full step where the gradient is near zero, and its step sizes follow the signs from
    then on, so there most, not all, elements agree."""
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
        ref = pdt.models.ConvNet().to(_dev())
        ropt = cls(ref.parameters(), **kw)
        step = GraphedTrainStep(ddp, crit, opt, batches[0], warmup=2, max_grad_norm=max_norm, accumulation_steps=k)
        assert step._riding and step.kernels_per_replay == 3 * k, step.kernels_per_replay
        if k > 1:
            assert step.accumulates_in_kernel
        steps0 = float(opt.state[next(iter(model.parameters()))]["step"])
        # the reference starts from where the engine's eager warm-up steps left the model and optimizer
        ref.load_state_dict(model.state_dict())
        ropt.load_state_dict(copy.deepcopy(opt.state_dict()))
        assert steps0 <= 4
        for i in range(12):
            x, t = batches[i % 4]
            params = list(model.parameters())
            snap = _snapshot(opt, params)
            step(x, t, inputs_ready=True)
            torch.cuda.synchronize()
            _expect(i, opt, params, [p.grad for p in params], snap)
            ropt.zero_grad()
            for j in range(k):
                (crit(ref(x[j * 100:(j + 1) * 100]), t[j * 100:(j + 1) * 100]) / k).backward()
            if max_norm is not None:
                torch.nn.utils.clip_grad_norm_(ref.parameters(), max_norm)
            ropt.step()
        torch.cuda.synchronize()
        for p, q in zip(model.parameters(), ref.parameters()):
            assert float(opt.state[p]["step"]) == float(ropt.state[q]["step"]) == steps0 + 12, "one step per replay"
            if name == "asgd":
                assert torch.equal(opt.state[p]["mu"], ropt.state[q]["mu"])
        keep = [(p, q) for (n, p), q in zip(model.named_parameters(), ref.parameters()) if n not in NOISE]
        a, b = _flat([p for p, _ in keep]), _flat([q for _, q in keep])
        if name == "rprop":
            far = ((a - b).abs() > 1e-3).double().mean().item()
            assert far < 0.1, far
        else:
            err = (a - b).abs().max().item() / b.abs().max().item()
            assert err < 2e-2, err
        opt.stop_riding()


@pytest.mark.gpu
# the replays run the update, never optimizer.step() itself, which torch's schedulers expect to see before their own step
@pytest.mark.filterwarnings("ignore:Detected call of `lr_scheduler.step\\(\\)` before `optimizer.step\\(\\)`")
@pytest.mark.parametrize("name", ["adamax", "adadelta", "asgd"])
def test_graphed_step_follows_a_learning_rate_schedule_and_refuses_a_new_fixed_key(name):
    """A LambdaLR that alternates lr between a decaying value and 0, stepped between ten replays: every replay within float64's bounds
    of its gradients at the scheduled lr, and ASGD's next eta formed from it.  Adamax and Adadelta leave the parameters bitwise
    unchanged at lr 0; ASGD does so one replay later, when the eta formed at lr 0 applies.  A changed fixed hyper-parameter is
    refused by the next replay."""
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
        frozen = 0
        for i in range(10):
            lr = opt.param_groups[0]["lr"]
            assert lr == (0.0 if i % 3 == 1 else kw["lr"] * (1.0 / (1 + i)))
            params = list(model.parameters())
            snap = _snapshot(opt, params)
            step(*xs[i % 4], inputs_ready=True)
            torch.cuda.synchronize()
            _expect(i, opt, params, [p.grad for p in params], snap)
            zero_step = lr == 0.0 if name != "asgd" else snap["eta"] == 0.0
            if zero_step:
                assert torch.equal(_flat(params), snap["p"]), (i, "a step at lr 0 changed the parameters")
                frozen += 1
            if name == "asgd":
                assert (float(opt.state[params[0]]["eta"]) == 0.0) == (lr == 0.0)
            sched.step()
        assert frozen >= 2
        key = cls._FIXED_KEYS[0]
        opt.param_groups[0][key] = _perturbed(opt.param_groups[0][key])
        with pytest.raises(RuntimeError, match=f"'{key}' of param_groups\\[0\\]"):
            step(*xs[0], inputs_ready=True)
        opt.stop_riding()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(RIDER_OPTS))
def test_checkpoint_resume_gives_the_uninterrupted_next_step(tmp_path, name):
    """Four steps, save_checkpoint, one more step; a fresh model and optimizer loaded from the checkpoint take the same fifth step
    bit for bit (step, and ASGD's eta and mu, come back to the device as fp32)."""
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
        for key in SCALARS[name]:
            assert opt2.state[p][key].is_cuda and opt2.state[p][key].dtype == torch.float32
    one_step(model2, opt2, 4)
    torch.cuda.synchronize()
    for p, q in zip(model.parameters(), model2.parameters()):
        assert torch.equal(p, q)
        for k in opt.state[p]:
            assert torch.equal(opt.state[p][k], opt2.state[q][k]), k
