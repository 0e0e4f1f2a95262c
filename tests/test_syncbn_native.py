"""SyncBatchNorm's native kernels against float64 on one GPU, with the other ranks of the process group emulated.

Both native SyncBatchNorm paths fall back to local batch norm in a world of one, so a fake process group stands in for rank r of a
world of R here: its in-line allreduce adds, in place, what the other ranks would contribute, taken from a float64 oracle of the
whole (concatenated) batch.  Rank r is thus checked against "every other rank exact":

* the generic path (``pdt.SyncBatchNorm`` on any N×C×… input): bn_stats_nchw_f64 → fp64 allreduce of (Σx, Σx², n) → bn_finalize
  (or the same arithmetic in Python) → bn_apply_nchw; backward bn_bwd_reduce_nchw → fp32 allreduce of (Σdy, Σdy·(x−μ)) →
  bn_bwd_apply_nchw;
* the ConvNet path (``convert_sync_batchnorm(ConvNet())``): conv5x5_fwd's zero-padded [2C+4] fp32 statistics are all-reduced before
  bn_relu_pool_fwd; backward all-reduces (Σdz, Σdz·x̂) of bn_relu_pool_bwd_reduce before bn_relu_pool_bwd_apply.

The oracle runs BatchNorm in float64 on the concatenated shards with one copy of every parameter per shard and the loss Σₖ Lₖ:
shard r's output and input gradient, and the gradients of its own parameter copies, are what rank r must produce.

Tolerances are first-order rounding bounds, with ε = 2⁻²⁴ (fp32) and u = 2⁻⁵³ (fp64).  A sum whose terms pass through at most d
additions is off by at most d·(unit roundoff)·Σ|terms|, whatever the order; ``_depth`` gives d for the kernels' per-channel sums,
and the torch-op fallback (PDT_SYNCBN_KERNELS=0, a control) is held to the order-free bound d = number of terms."""
import pytest
import torch
import torch.nn.functional as F

import pytorch_distributed_train_b200 as pdt
from pytorch_distributed_train_b200 import distributed as dist
from pytorch_distributed_train_b200 import ops
from pytorch_distributed_train_b200.ops import functional as OF

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -24   # fp32 unit roundoff
U64 = 2.0 ** -53   # fp64 unit roundoff
BN_EPS = 1e-5


def dev():
    return torch.device("cuda", 0)


# ---- the emulated process group -------------------------------------------------------------------------------------------------
class _FakeComm:
    """Rank r's in-line SUM allreduce: checks the call against the next expected one and adds the other ranks' part in place."""

    def __init__(self):
        self.expected = []   # (what, dtype, length, the other ranks' sum, first pad index or None)
        self.calls = []

    def allreduce_inline(self, t, op, postscale):
        assert self.expected, f"unexpected allreduce of {t.numel()} x {t.dtype}"
        what, dtype, length, others, pad_from = self.expected.pop(0)
        assert op == dist.ReduceOp.SUM and postscale == 1.0, (what, op, postscale)
        assert t.is_cuda and t.is_contiguous() and t.dtype == dtype and t.numel() == length, (what, t.dtype, t.numel(), dtype, length)
        if pad_from is not None:
            assert bool((t[pad_from:] == 0).all()), (what, "pad entries are not zero", t[pad_from:].tolist())
        t.add_(others.to(device=t.device, dtype=t.dtype))
        self.calls.append(what)


class _FakeGroup:
    """Rank r of a world of R: ``size()``, ``is_cuda`` and ``comm`` are all that either SyncBatchNorm path touches."""
    is_cuda = True

    def __init__(self, world):
        self.world = world
        self.comm = _FakeComm()

    def size(self):
        return self.world


@pytest.fixture
def fake_dist(monkeypatch):
    """Both paths ask ``distributed.is_initialized()`` before they look at the group; nothing global is set up."""
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    return monkeypatch


# ---- summation depth, inputs and the float64 oracle of the generic path ----------------------------------------------------------
def _depth(total, C):
    """Longest chain of additions a term meets in bn_stats_nchw_f64_kernel / bn_bwd_reduce_nchw_kernel: a thread's serial loop
    over its share of one of S slices of the channel (S from bn_slices in ops_simt.cu), 5 shuffle levels, 8 warps, S slices."""
    if total == 0:
        return 0
    S = max(1, min(max(1, total // 2048), max(1, 592 // C)))
    return -(-(-(-total // S)) // 256) + 5 + 8 + S


def _dims(x):
    return [0] + list(range(2, x.dim()))


def _bshape(x):
    return [1, -1] + [1] * (x.dim() - 2)


def _inputs(cond, N, C, spatial, gen):
    z = torch.randn((N, C) + tuple(spatial), device=dev(), generator=gen)
    shp = [1, -1] + [1] * len(spatial)
    if cond == "well":
        mean = torch.randn(C, device=dev(), generator=gen)
        std = torch.rand(C, device=dev(), generator=gen) * 1.5 + 0.5
    else:   # mean ≫ spread: μ = ±100 or ±1000 (up to 10 % more), σ = 0.1
        sign = 1.0 - 2.0 * (torch.arange(C, device=dev()) % 2)
        mean = sign * {"mu100": 100.0, "mu1000": 1000.0}[cond] * (1 + 0.1 * torch.rand(C, device=dev(), generator=gen))
        std = torch.full((C,), 0.1, device=dev())
    return z * std.view(shp) + mean.view(shp)


class _Oracle:
    """float64 BatchNorm over the concatenated shards, one copy of γ and β per shard, loss Σₖ ⟨yₖ, dyₖ⟩."""

    def __init__(self, shards, weight, bias, dys):
        C = shards[0].shape[1]
        xs = [s.double().requires_grad_() for s in shards]
        x = torch.cat(xs)
        dims, shp = _dims(x), _bshape(x)
        self.shp = shp
        mean, var = x.mean(dims), x.var(dims, unbiased=False)
        invstd = (var + BN_EPS).rsqrt()
        ws = [None if weight is None else weight.double().requires_grad_() for _ in shards]
        bs = [None if bias is None else bias.double().requires_grad_() for _ in shards]
        ys = []
        for xk, wk, bk in zip(xs, ws, bs):
            yk = (xk - mean.view(shp)) * invstd.view(shp)
            yk = yk * wk.view(shp) if wk is not None else yk
            yk = yk + bk.view(shp) if bk is not None else yk
            ys.append(yk)
        sum((yk * dk.double()).sum() for yk, dk in zip(ys, dys)).backward()
        self.C, self.N = C, x.numel() // C
        self.x64 = x.detach()
        self.mean, self.var, self.invstd = mean.detach(), var.detach(), invstd.detach()
        self.weight = weight
        self.y = [yk.detach() for yk in ys]
        self.dx = [xk.grad for xk in xs]
        self.dw = [None if wk is None else wk.grad for wk in ws]
        self.db = [None if bk is None else bk.grad for bk in bs]
        self.dy = [dk.double() for dk in dys]
        self.ex2 = (self.x64 * self.x64).mean(dims)
        self.eabs = self.x64.abs().mean(dims)
        # per-shard (Σx, Σx², n, pad), shifted by c = fl32(μ) so that each is accurate to a few roundings of its result whatever
        # μ/σ: the other ranks are exact
        c = self.mean.float().double()
        self.fwd_sums, self.local_abs = [], []
        for s in shards:
            sd = s.double()
            d = sd - c.view(shp)
            n = s.numel() // C
            s1 = d.sum(dims)
            self.fwd_sums.append(torch.cat([n * c + s1, n * c * c + 2 * c * s1 + (d * d).sum(dims), d.new_tensor([float(n), 0.0])]))
            self.local_abs.append((sd.abs().sum(dims), (sd * sd).sum(dims)))
        # per-shard (Σdy, Σdy·(x−μ)) and the magnitudes the fp32 bounds need
        self.a = [s.double() - self.mean.view(shp) for s in shards]
        self.bwd_sums = [torch.cat([dk.sum(dims), (dk * ak).sum(dims)]) for dk, ak in zip(self.dy, self.a)]
        self.dy_abs = [dk.abs().sum(dims) for dk in self.dy]
        self.dya_abs = [(dk * ak).abs().sum(dims) for dk, ak in zip(self.dy, self.a)]

    @staticmethod
    def others(per_shard, r):
        return sum(s for k, s in enumerate(per_shard) if k != r)

    def stat_bounds(self, d_stats):
        """Bounds on fl32(μ) and on the errors of var and fl32(invstd) when rank r's fp64 sums are d_stats additions deep (the
        other ranks' part and the exchange add one each): δΣ ≤ (d+2)·u·Σ|·|, so |δμ| ≤ (d+2)·u·E|x| + ε·|μ| and
        |δvar| ≤ (d+4)·u·(E[x²] + 2|μ|·E|x|).  invstd = (var+eps)^-½ carries half the relative error of var+eps, plus the fp64
        rsqrt and the rounding to fp32."""
        tol_mean = (d_stats + 2) * U64 * self.eabs + EPS * self.mean.abs()
        dvar = (d_stats + 4) * U64 * (self.ex2 + 2 * self.mean.abs() * self.eabs)
        rel_is = 0.5 * dvar / (self.var + BN_EPS) + 2 * EPS
        return tol_mean, dvar, rel_is


def _assert_within(got, ref, tol, what):
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    err = (got.double() - ref).abs()
    bad = ~(err <= tol)
    assert not bool(bad.any()), (what, int(bad.sum()), (err / tol.clamp_min(1e-300)).max().item())


def _check_y(o, r, y, tol_mean, rel_is):
    """y = fl(fl(fl(x − fl μ)·fl invstd)·γ + β): x − μ is exact by Sterbenz when |μ| ≫ σ, so the error is the mean's rounding
    carried through, |γ|·invstd·|δμ|, plus invstd's relative error and three roundings on |x̂γ|, plus two ulp of y."""
    shp = o.shp
    g = o.weight.double().abs().view(shp) if o.weight is not None else 1.0
    is_ = o.invstd.view(shp)
    xhat_g = (o.a[r] * is_).abs() * g
    tol = g * is_ * tol_mean.view(shp) + xhat_g * (rel_is.view(shp) + 4 * EPS) + 4 * EPS * o.y[r].abs()
    _assert_within(y, o.y[r], tol, "y")


def _check_dx(o, r, dx, tol_mean, rel_is, d_red):
    """dx = γ·invstd·(dy − M₁ − (x − fl μ)·invstd²·M₂) with M₁ = Σdy/n and M₂ = Σdy·(x−μ)/n over the group.  Rank r's part of
    each sum is d_red fp32 additions deep (the other ranks' rounding, the exchange and the division add three), and its
    Σdy·(x − fl μ) differs from Σdy·(x−μ) by |δμ|·Σ|dy|.  Each term of the bracket is off by its inputs' errors, invstd enters
    three times in the last term and once outside, and four roundings act on the bracket, three on the product."""
    shp = o.shp
    n = o.N
    dy_abs, dya_abs = sum(o.dy_abs).view(shp), sum(o.dya_abs).view(shp)
    sums = sum(o.bwd_sums)
    m1, m2 = (sums[:o.C] / n).abs().view(shp), (sums[o.C:] / n).abs().view(shp)
    tm, ri, is_ = tol_mean.view(shp), rel_is.view(shp), o.invstd.view(shp)
    e1 = (d_red + 3) * EPS * dy_abs / n + EPS * m1
    e2 = ((d_red + 4) * EPS * dya_abs + tm * dy_abs) / n + EPS * m2
    g = o.weight.double().abs().view(shp) if o.weight is not None else 1.0
    a = o.a[r].abs()
    third = a * is_ * is_ * m2
    bracket = 4 * EPS * (o.dy[r].abs() + m1 + third) + e1 + a * is_ * is_ * e2 + (tm + EPS * a) * is_ * is_ * m2 + 3 * ri * third
    tol = g * is_ * bracket + o.dx[r].abs() * (ri + 3 * EPS)
    _assert_within(dx, o.dx[r], tol, "dx")


def _check_param_grads(o, r, dw, db, tol_mean, rel_is, d_red):
    """dβ = Σdy and dγ = Σdy·(x − fl μ)·invstd over the local shard only (fp32 sums d_red deep; DDP sums them across ranks)."""
    tol_b = d_red * EPS * o.dy_abs[r]
    _assert_within(db, o.db[r], tol_b, "dbeta")
    tol_w = o.invstd * ((d_red + 2) * EPS * o.dya_abs[r] + tol_mean * o.dy_abs[r]) + o.dw[r].abs() * (rel_is + EPS)
    _assert_within(dw, o.dw[r], tol_w, "dgamma")


# ---- generic path cases ---------------------------------------------------------------------------------------------------------
# (id, C, spatial dims, per-rank batch sizes, rank under test)
GENERIC = [
    ("resnet_64x112", 64, (112, 112), (4, 5), 0),        # ResNet-18's BatchNorms at 4 images per rank
    ("resnet_64x56", 64, (56, 56), (4, 3), 0),
    ("resnet_128x28", 128, (28, 28), (4, 6), 0),
    ("resnet_256x14", 256, (14, 14), (4, 4), 1),
    ("resnet_512x7", 512, (7, 7), (4, 2), 0),
    ("bn1d_NC", 48, (), (16, 9), 1),                     # BatchNorm1d [N, C] and [N, C, L]
    ("bn1d_NCL", 24, (50,), (5, 3), 0),
    ("bn3d_NCDHW", 8, (4, 6, 5), (3, 2), 1),
    ("c1_n2047", 1, (), (2047, 9), 0),                   # N·HW just below and above 2048·S, S = 1, 2 and the cap 592
    ("c1_n2049", 1, (), (2049, 9), 0),
    ("c1_n4095", 1, (), (4095, 9), 0),
    ("c1_n4097", 1, (), (4097, 9), 0),
    ("c1_n1212415", 1, (), (2048 * 592 - 1, 9), 0),
    ("c1_n1212417", 1, (), (2048 * 592 + 1, 9), 0),
    ("c600_n2047", 600, (), (2047, 5), 0),               # C > 592: one slice per channel
    ("c600_n2049", 600, (), (2049, 5), 0),
    ("c2048_n2047", 2048, (), (2047, 3), 0),
    ("c2048_n2049", 2048, (), (2049, 3), 0),
    ("world8", 64, (14, 14), (4, 3, 5, 1, 0, 7, 2, 4), 3),
    ("world8_local_empty", 64, (14, 14), (0, 3, 5, 1, 0, 7, 2, 4), 0),
    ("world8_others_empty", 32, (9, 7), (6, 0, 0, 0, 0, 0, 0, 0), 0),
    ("world2_local_empty", 16, (5, 5), (3, 0), 1),
    ("world2_other_empty", 16, (5, 5), (3, 0), 0),
]
CONDS = ["well", "mu100", "mu1000"]
MASKS = [15, 31, 0]   # the default kernels; plus the fused bn_finalize; the torch-op fallback (control)


def _case_data(case, cond, seed=0):
    _, C, spatial, ns, r = case
    gen = torch.Generator(device=dev()).manual_seed(1000 + seed)
    x = _inputs(cond, sum(ns), C, spatial, gen)
    dy = torch.randn(x.shape, device=dev(), generator=gen)
    return list(x.split(list(ns))), list(dy.split(list(ns))), r


def _queue(o, group, r, needs_dx):
    C = o.C
    group.comm.expected.append(("forward", torch.float64, 2 * C + 2, o.others(o.fwd_sums, r), 2 * C + 1))
    if needs_dx:
        group.comm.expected.append(("backward", torch.float32, 2 * C, o.others(o.bwd_sums, r), None))


def _run_generic(case, cond, mask, mp, affine=True, momentum=0.1, track=True, steps=1, needs_dx=True):
    mp.setenv("PDT_SYNCBN_KERNELS", str(mask))
    _, C, spatial, ns, r = case
    group = _FakeGroup(len(ns))
    mod = pdt.SyncBatchNorm(C, momentum=momentum, affine=affine, track_running_stats=track, process_group=group).to(dev())
    gen = torch.Generator(device=dev()).manual_seed(7)
    if affine:
        with torch.no_grad():
            mod.weight.copy_((torch.rand(C, device=dev(), generator=gen) + 0.5) * (1.0 - 2.0 * (torch.arange(C, device=dev()) % 3 == 0)))
            mod.bias.copy_(torch.randn(C, device=dev(), generator=gen) * 0.1)
    weight = mod.weight.detach().clone() if affine else None
    bias = mod.bias.detach().clone() if affine else None
    if track:
        with torch.no_grad():
            mod.running_mean.normal_(0.0, 0.1, generator=gen)
            mod.running_var.uniform_(0.5, 1.5, generator=gen)
        rm, rv = mod.running_mean.double().clone(), mod.running_var.double().clone()
        err_m, err_v = torch.zeros_like(rm), torch.zeros_like(rv)
    for step in range(steps):
        shards, dys, r = _case_data(case, cond, seed=step)
        o = _Oracle(shards, weight, bias, dys)
        _queue(o, group, r, needs_dx)
        total = shards[r].numel() // C
        d_stats = _depth(total, C) if mask & 1 else total
        d_red = _depth(total, C) if mask & 4 else total
        tol_mean, dvar, rel_is = o.stat_bounds(d_stats)
        xr = shards[r].clone().requires_grad_(needs_dx)
        if affine:
            mod.weight.grad = mod.bias.grad = None
        y = mod(xr)
        y.backward(dys[r])
        assert group.comm.expected == [], group.comm.expected
        assert y.dtype == torch.float32
        _check_y(o, r, y, tol_mean, rel_is)
        if needs_dx:
            _check_dx(o, r, xr.grad, tol_mean, rel_is, d_red)
        else:
            assert xr.grad is None
        if affine:
            _check_param_grads(o, r, mod.weight.grad, mod.bias.grad, tol_mean, rel_is, d_red)
        if track:
            # nn.BatchNorm's update in float64 on the whole batch (momentum None: the cumulative average, 1/t at step t).  Each fp32
            # step ρ' = (1−m)·ρ + m·s rounds four times on |ρ| + |s| and carries m times the statistic's error; the errors of
            # earlier steps shrink by (1 − m) ≤ 1.
            m = momentum if momentum is not None else 1.0 / (step + 1)
            n = o.N
            unbiased = o.var * n / (n - 1)
            err_m += 4 * EPS * (rm.abs() + o.mean.abs()) + m * tol_mean
            err_v += 4 * EPS * (rv.abs() + unbiased) + m * (dvar * n / (n - 1) + 2 * EPS * unbiased)
            with torch.no_grad():
                F.batch_norm(o.x64, rm, rv, None, None, True, m, BN_EPS)
            _assert_within(mod.running_mean, rm, err_m, "running_mean")
            _assert_within(mod.running_var, rv, err_v, "running_var")
            assert int(mod.num_batches_tracked) == step + 1
        else:
            assert mod.running_mean is None and mod.running_var is None
    assert group.comm.calls == (["forward", "backward"] if needs_dx else ["forward"]) * steps


@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("cond", CONDS)
@pytest.mark.parametrize("case", GENERIC, ids=[c[0] for c in GENERIC])
def test_generic_syncbn_matches_float64(case, cond, mask, fake_dist):
    _run_generic(case, cond, mask, fake_dist)


OPTION_CASES = [GENERIC[1], GENERIC[5], GENERIC[7], GENERIC[19]]


@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("cond", ["well", "mu1000"])
@pytest.mark.parametrize("case", OPTION_CASES, ids=[c[0] for c in OPTION_CASES])
@pytest.mark.parametrize("opt", ["affine_false", "momentum_none_3_steps", "no_running_stats", "no_dx"])
def test_generic_syncbn_options_match_float64(opt, case, cond, mask, fake_dist):
    kw = {"affine_false": dict(affine=False), "momentum_none_3_steps": dict(momentum=None, steps=3),
          "no_running_stats": dict(track=False), "no_dx": dict(needs_dx=False)}[opt]
    _run_generic(case, cond, mask, fake_dist, **kw)


# ---- the generic kernels called directly ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("cond", CONDS)
@pytest.mark.parametrize("case", GENERIC, ids=[c[0] for c in GENERIC])
def test_generic_bn_kernels_direct_match_float64(case, cond):
    """ops.bn_local_stats / bn_finalize / bn_apply / bn_backward_reduce / bn_backward_apply on rank r's shard, the other ranks'
    sums added as the allreduce would; every result the same bit for bit on a second call (each fold runs in a fixed order)."""
    C = case[1]
    shards, dys, r = _case_data(case, cond)
    gen = torch.Generator(device=dev()).manual_seed(11)
    w = torch.rand(C, device=dev(), generator=gen) + 0.5
    b = torch.randn(C, device=dev(), generator=gen) * 0.1
    o = _Oracle(shards, w, b, dys)
    x, dy = shards[r].contiguous(), dys[r].contiguous()
    total = x.numel() // C
    d = _depth(total, C)

    st = ops.bn_local_stats(x)
    assert st.dtype == torch.float64 and st.numel() == 2 * C + 2
    assert torch.equal(st, ops.bn_local_stats(x))
    assert st[2 * C].item() == total and st[2 * C + 1].item() == 0.0
    s_abs, s2 = o.local_abs[r]
    _assert_within(st[:C], o.fwd_sums[r][:C], (d + 1) * U64 * s_abs, "Σx")
    _assert_within(st[C:2 * C], o.fwd_sums[r][C:2 * C], (d + 1) * U64 * s2, "Σx²")

    tol_mean, dvar, rel_is = o.stat_bounds(d)
    if cond == "mu1000":
        # μ/σ = 10⁴: the derived bound on invstd stays near 1e-6 for folds a few dozen additions deep and reaches 1.1e-5 at 592 slices
        # (613 deep); fp32 sums of the same terms would be off by about 2⁻²⁴·μ²/σ² ≈ 6, relative
        assert rel_is.max().item() < (1.5e-6 if d < 64 else 2e-5), (d, rel_is.max().item())
    full = st + o.others(o.fwd_sums, r)
    rm0 = torch.randn(C, device=dev(), generator=gen) * 0.1
    rv0 = torch.rand(C, device=dev(), generator=gen) + 0.5
    rm, rv, rm2, rv2 = rm0.clone(), rv0.clone(), rm0.clone(), rv0.clone()
    mean, invstd, count = ops.bn_finalize(full, C, BN_EPS, 0.1, rm, rv)
    mean2, invstd2, count2 = ops.bn_finalize(full, C, BN_EPS, 0.1, rm2, rv2)
    assert torch.equal(mean, mean2) and torch.equal(invstd, invstd2) and torch.equal(rm, rm2) and torch.equal(rv, rv2)
    assert count.item() == o.N
    _assert_within(mean, o.mean, tol_mean, "mean")
    _assert_within(invstd, o.invstd, o.invstd * rel_is, "invstd")
    n = o.N
    unbiased = o.var * n / (n - 1)
    rm_ref, rv_ref = rm0.double().clone(), rv0.double().clone()
    F.batch_norm(o.x64, rm_ref, rv_ref, None, None, True, 0.1, BN_EPS)
    _assert_within(rm, rm_ref, 4 * EPS * (rm0.double().abs() + o.mean.abs()) + 0.1 * tol_mean, "running_mean")
    _assert_within(rv, rv_ref, 4 * EPS * (rv0.double().abs() + unbiased) + 0.1 * (dvar * n / (n - 1) + 2 * EPS * unbiased),
                   "running_var")

    y = ops.bn_apply(x, mean, invstd, w, b)
    assert torch.equal(y, ops.bn_apply(x, mean, invstd, w, b))
    _check_y(o, r, y, tol_mean, rel_is)

    red = ops.bn_backward_reduce(dy, x, mean, invstd)
    assert torch.equal(red, ops.bn_backward_reduce(dy, x, mean, invstd))
    assert red.numel() == 4 * C and torch.equal(red[3 * C:], red[:C])
    _assert_within(red[:C], o.bwd_sums[r][:C], d * EPS * o.dy_abs[r], "Σdy")
    _assert_within(red[C:2 * C], o.bwd_sums[r][C:], (d + 2) * EPS * o.dya_abs[r] + tol_mean * o.dy_abs[r], "Σdy·(x−μ)")
    _check_param_grads(o, r, red[2 * C:3 * C], red[3 * C:], tol_mean, rel_is, d)

    sums = red[:2 * C] + o.others(o.bwd_sums, r).float()
    dx = ops.bn_backward_apply(dy, x, mean, invstd, w, sums[:C] / n, sums[C:] / n)
    assert torch.equal(dx, ops.bn_backward_apply(dy, x, mean, invstd, w, sums[:C] / n, sums[C:] / n))
    _check_dx(o, r, dx, tol_mean, rel_is, d)


# ---- the ConvNet path -----------------------------------------------------------------------------------------------------------
def _float64_twin(net):
    ref = pdt.models.ConvNet(num_classes=net.fc.out_features, fused=False).to(dev())
    ref.load_state_dict(net.state_dict())
    return ref.double()


def _convnet_oracle(twins, xs, ts):
    """The fused=False float64 twin, one per shard, with each BatchNorm's statistics taken over all shards; loss Σₖ Lₖ.  Returns
    per layer the per-shard conv outputs y, the BN outputs z (their .grad = dz), the global mean / invstd and the running
    statistics nn.BatchNorm2d would hold; and the per-shard logits and losses."""
    acts = [x.double() for x in xs]
    layers = {}
    for l in (1, 2):
        convs = [getattr(tw, f"layer{l}")[0] for tw in twins]
        bns = [getattr(tw, f"layer{l}")[1] for tw in twins]
        ys = [cv(a) for cv, a in zip(convs, acts)]
        yall = torch.cat(ys)
        mean, var = yall.mean((0, 2, 3)), yall.var((0, 2, 3), unbiased=False)
        invstd = (var + bns[0].eps).rsqrt()
        v = lambda t: t.view(1, -1, 1, 1)  # noqa: E731
        zs = []
        for y, bn in zip(ys, bns):
            z = (y - v(mean)) * v(invstd) * v(bn.weight) + v(bn.bias)
            z.retain_grad()
            zs.append(z)
        acts = [F.max_pool2d(F.relu(z), 2, 2) for z in zs]
        rm, rv = bns[0].running_mean.clone(), bns[0].running_var.clone()
        with torch.no_grad():
            F.batch_norm(yall, rm, rv, None, None, True, bns[0].momentum, bns[0].eps)
        layers[l] = dict(ys=ys, zs=zs, mean=mean, invstd=invstd, rm=rm, rv=rv, gamma=bns[0].weight.detach())
    logits = [tw.fc(a.reshape(a.shape[0], -1)) for tw, a in zip(twins, acts)]
    losses = [F.cross_entropy(lg, t) for lg, t in zip(logits, ts)]
    sum(losses).backward()
    return layers, logits, losses


def _norm_close(got, ref, what, scale=None):
    # TF32 (conv2 forward and dgrad, 10-bit mantissa): test_kernel_edges.py's policy, measured over the whole tensor, relative to
    # the magnitude of the terms the result is made of (`scale`, by default the result itself)
    err, norm = (got.double() - ref).norm().item(), (ref if scale is None else scale).norm().item()
    assert err <= 3e-2 * norm + 1e-4 * ref.numel() ** 0.5, (what, err, norm)


def _conv_bias_scale(layer, r):
    """A conv bias in front of a SyncBatchNorm gets rank r's Σdy = γ·invstd·(Σdz − n_r·M₁ − M₂·Σx̂) over its own shard, M₁ and M₂
    the group means of dz and dz·x̂: a difference of nearly equal terms, whose TF32 noise scales with the terms' magnitudes."""
    v = lambda t: t.detach().view(1, -1, 1, 1)  # noqa: E731
    xh = [(y.detach() - v(layer["mean"])) * v(layer["invstd"]) for y in layer["ys"]]
    dz = [z.grad for z in layer["zs"]]
    n = sum(d.numel() for d in dz) // dz[0].shape[1]
    m1 = sum(d.sum((0, 2, 3)) for d in dz) / n
    m2 = sum((d * x).sum((0, 2, 3)) for d, x in zip(dz, xh)) / n
    n_r = dz[r].numel() // dz[r].shape[1]
    terms = dz[r].abs().sum((0, 2, 3)) + n_r * m1.abs() + m2.abs() * xh[r].abs().sum((0, 2, 3))
    return layer["gamma"].abs() * layer["invstd"].detach() * terms


def _grad_scale(name, layers, r):
    """The magnitude of the terms each gradient is summed from, where that differs from the gradient itself: the local sums
    dβ = Σdz and dγ = Σdz·x̂ of a small shard cancel as much as the conv biases' do."""
    if name.endswith(".0.bias"):
        return _conv_bias_scale(layers[int(name[5])], r)
    if name.endswith(".1.bias") or name.endswith(".1.weight"):
        L = layers[int(name[5])]
        dz = L["zs"][r].grad
        if name.endswith(".1.bias"):
            return dz.abs().sum((0, 2, 3))
        xh = (L["ys"][r].detach() - L["mean"].detach().view(1, -1, 1, 1)) * L["invstd"].detach().view(1, -1, 1, 1)
        return (dz * xh).abs().sum((0, 2, 3))
    return None


@pytest.mark.parametrize("ns,r", [((37, 63), 0), ((37, 63), 1), ((1, 99), 0), ((1, 99), 1), ((10, 40, 25, 25), 2), ((3, 50, 1, 46), 2)])
def test_convnet_syncbn_matches_float64(ns, r, fake_dist):
    torch.manual_seed(5)
    gen = torch.Generator(device=dev()).manual_seed(9)
    group = _FakeGroup(len(ns))
    net = pdt.SyncBatchNorm.convert_sync_batchnorm(pdt.models.ConvNet(), process_group=group).to(dev())
    assert type(net.layer1[1]) is pdt.SyncBatchNorm and type(net.layer2[1]) is pdt.SyncBatchNorm
    twins = [_float64_twin(net) for _ in ns]
    x = torch.rand(sum(ns), 1, 28, 28, device=dev(), generator=gen)
    t = torch.randint(0, 10, (sum(ns),), device=dev(), generator=gen)
    xs, ts = list(x.split(list(ns))), list(t.split(list(ns)))
    layers, logits_ref, losses = _convnet_oracle(twins, xs, ts)

    others = lambda per: sum(p for k, p in enumerate(per) if k != r)  # noqa: E731
    for l, C in ((1, 16), (2, 32)):
        ys = [y.detach() for y in layers[l]["ys"]]
        fwd = [torch.cat([y.sum((0, 2, 3)), (y * y).sum((0, 2, 3)), y.new_tensor([float(y.numel() // C), 0.0, 0.0, 0.0])]) for y in ys]
        group.comm.expected.append((f"layer{l} forward", torch.float32, 2 * C + 4, others(fwd), 2 * C + 1))
    for l in (2, 1):
        L = layers[l]
        xhat = [(y.detach() - L["mean"].detach().view(1, -1, 1, 1)) * L["invstd"].detach().view(1, -1, 1, 1) for y in L["ys"]]
        bwd = [torch.cat([z.grad.sum((0, 2, 3)), (z.grad * xh).sum((0, 2, 3))]) for z, xh in zip(L["zs"], xhat)]
        group.comm.expected.append((f"layer{l} backward", torch.float32, 2 * L["mean"].numel(), others(bwd), None))

    xr = xs[r].contiguous()
    assert not OF.fused_convnet_ok(xr, net)   # SyncBatchNorm takes the per-op kernels
    logits = net(xr)
    loss = pdt.nn.CrossEntropyLoss()(logits, ts[r])
    loss.backward()
    assert group.comm.calls == ["layer1 forward", "layer2 forward", "layer2 backward", "layer1 backward"], group.comm.calls
    assert group.comm.expected == []

    # conv2 runs in TF32: loss, logits and gradients at test_kernel_edges.py's TF32 level
    assert abs(loss.item() - losses[r].item()) < 2e-3, (loss.item(), losses[r].item())
    _norm_close(logits.detach(), logits_ref[r].detach(), "logits")
    for (name, p), (_, q) in zip(net.named_parameters(), twins[r].named_parameters()):
        _norm_close(p.grad, q.grad, name, _grad_scale(name, layers, r))
    for l in (1, 2):
        bn = getattr(net, f"layer{l}")[1]
        assert int(bn.num_batches_tracked) == 1
        # batch statistics of the TF32 conv2 output (test_kernel_edges.py)
        for got, ref, what in ((bn.running_mean, layers[l]["rm"], "running_mean"), (bn.running_var, layers[l]["rv"], "running_var")):
            assert torch.allclose(got.double(), ref, atol=2e-3, rtol=1e-3), (l, what, (got.double() - ref).abs().max().item())
