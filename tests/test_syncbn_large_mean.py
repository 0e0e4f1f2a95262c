"""The ConvNet's SyncBatchNorm statistics where a channel's mean dwarfs its spread, against float64.

Under ``convert_sync_batchnorm`` the ConvNet runs the per-op kernels, and each rank sends its layer's batch statistics through one
all-reduce before bn_relu_pool_fwd normalises with the group's mean and variance.  Those sums must not lose the variance's digits
when |mean| ≫ std (a conv bias in front of a BatchNorm has no true gradient and stays where it was initialised or loaded): each
rank forms fp64 [Σy = n·mean, Σy² = M2 + n·mean², n, 0] from its centred fold (conv5x5_fwd fp64_sums), and the group's mean and
variance are taken in fp64.  fp32 Σy²/n − mean² would be off by about 2⁻²⁴·(mean/std)² relative.

As in test_syncbn_native.py, one GPU plays rank r of the group and a fake process group adds, in place, what the other ranks
would contribute.  Here that contribution is computed in float64 from the other shards' conv outputs produced by the same kernel
call the path makes, and the rank's own conv output is recorded from the path, so the statistics are compared with float64
statistics of exactly the values the group normalises (TF32 rounding in conv2 stays out of it).  The conv biases are set to r
times each channel's spread for r up to 3000.  The statistics are held to the one-GPU contract of test_bn_large_mean.py.
Covered: one layer at a time (both convolutions, uneven and one-image shards), a whole training step of the ConvNet against the
float64 oracle followed by an eval forward with the updated running statistics, and the same on two real ranks with DDP and the
graph-captured step."""
import pytest
import torch
import torch.nn.functional as F

import pytorch_distributed_train_b200 as pdt
from pytorch_distributed_train_b200 import _C
from pytorch_distributed_train_b200 import ops
from pytorch_distributed_train_b200.ops import functional as OF
from mp_helpers import run_ranks
from test_bn_large_mean import _offset_biases, _spread
from test_syncbn_native import _FakeGroup, _convnet_oracle, _float64_twin, _grad_scale, _norm_close, fake_dist  # noqa: F401

pytestmark = pytest.mark.gpu

RATIOS = [1, 30, 300, 3000]
# (per-rank batch sizes, rank under test): uneven shards from either side, a one-image rank, and a rank among four
SHARDS = [((37, 63), 0), ((37, 63), 1), ((1, 99), 0), ((3, 50, 1, 46), 2)]
# the forward exchange of the per-op SyncBatchNorm path: its dtype, the kernel call that produces it and its pad entries
WIRE_DTYPE, WIRE_PAD, PATH_STATS = torch.float64, 1, dict(fp64_sums=True)


def dev():
    return torch.device("cuda", 0)


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


class _Recorder:
    """Stands in for the extension module inside ops.functional and keeps every conv output the path computes."""

    def __init__(self):
        self.ys = []

    def __getattr__(self, name):
        return getattr(_C, name)

    def conv5x5_fwd(self, *args, **kw):
        y, stats = _C.conv5x5_fwd(*args, **kw)
        self.ys.append(y)
        return y, stats


def _conv_y(xh, w, b):
    """y of the kernel call the SyncBatchNorm path makes, checked to repeat bit for bit (the tests rely on the path computing the
    same y for the same shard)."""
    y = _C.conv5x5_fwd(xh, w, b, True, **PATH_STATS)[0]
    assert torch.equal(y, _C.conv5x5_fwd(xh, w, b, True, **PATH_STATS)[0])
    return y


def _wire(y, C):
    """One rank's part of the forward exchange, exact in float64: [Σy, Σy², n] and the pad entries."""
    v = y.double().reshape(-1, C)
    return torch.cat([v.sum(0), (v * v).sum(0), v.new_tensor([float(v.shape[0])] + [0.0] * WIRE_PAD)])


def _queue_forward(group, what, ys, r, C):
    others = sum(_wire(y, C) for k, y in enumerate(ys) if k != r)
    group.comm.expected.append((what, WIRE_DTYPE, 2 * C + 1 + WIRE_PAD, others, 2 * C + 1))


def _check_running(rm, rv, rm0, rv0, m, v, what):
    """The running statistics after one update with momentum m from (rm0, rv0), against float64 statistics of the whole group's
    conv outputs v [N, C]: test_bn_large_mean.py's contract, the mean within 1e-5·std + 2⁻²²·|mean| and the variance within
    2e-5 + 2⁻²⁴·|mean|/std relative (what fp32 values near |mean| cost a centred fold)."""
    N = v.shape[0]
    mean, var = v.mean(0), v.var(0, unbiased=False)
    std = var.sqrt()
    var_tol = 2e-5 + 2.0 ** -24 * mean.abs() / std
    ref_rm = (1 - m) * rm0 + m * mean
    err = ((rm.double() - ref_rm).abs() / (1e-5 * std + 2.0 ** -22 * (ref_rm.abs() + mean.abs()))).max().item()
    assert err <= 1, (what, "running mean (share of the tolerance)", err)
    ref_rv = (1 - m) * rv0 + m * var * N / (N - 1)
    rel = ((rv.double() - ref_rv).abs() / ref_rv)
    assert (rel / var_tol).max().item() <= 1, (what, "running var: relative error", rel.max().item(), "tolerance",
                                               var_tol[rel.argmax()].item())
    return mean, var, var_tol


def _check_out(out, y, mean, var, var_tol, gamma, beta, eps):
    """The BN + ReLU + pool output (NCHW) against float64 BatchNorm of the kernel's own y (NHWC) with the group's statistics.  The mean
    and variance errors allowed above pass through γ·invstd and x̂·γ; fmaf(y, γ·invstd, β − mean·γ·invstd) rounds terms of size
    γ·invstd·|y| a few times (2⁻²¹ of them: y ≈ mean, so that is 2⁻²¹·|mean|/std·γ), and ReLU and the 2×2 max move no error up."""
    y = y.double()
    g, b = gamma.double(), beta.double()
    invstd = (var + eps).rsqrt()
    xhat = (y - mean) * invstd
    z = xhat * g + b
    tol_mean = 1e-5 * var.sqrt() + 2.0 ** -22 * mean.abs()
    tol = g.abs() * invstd * tol_mean + (xhat * g).abs() * var_tol + 2.0 ** -21 * (g.abs() * invstd * y.abs() + b.abs()) + 2.0 ** -21 * z.abs()
    ref = F.max_pool2d(F.relu(z).permute(0, 3, 1, 2), 2, 2)
    tol = F.max_pool2d(tol.permute(0, 3, 1, 2), 2, 2)
    err = (out.double() - ref).abs()
    assert bool((err <= tol).all()), ("output", (err / tol).max().item(), err.max().item())


# ---- one layer at a time ----------------------------------------------------------------------------------------------------------
def _layer_case(layer, ns, ratio, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    cin, C, H = (1, 16, 28) if layer == 1 else (16, 32, 14)
    x = torch.rand(sum(ns), cin, H, H, generator=g).to(dev())
    w = (torch.randn(C, cin, 5, 5, generator=g) * (0.2 if layer == 1 else 0.05)).to(dev())
    b = (ratio * _spread(F.conv2d(x.double(), w.double(), padding=2))).float()
    gamma = (1.0 + torch.randn(C, generator=g) * 0.1).to(dev())
    beta = (torch.randn(C, generator=g) * 0.1).to(dev())
    return list(x.split(list(ns))), w, b, gamma, beta, C


def _run_layer(xs, w, b, gamma, beta, C, r, momentum, mp):
    group = _FakeGroup(len(xs))
    conv = torch.nn.Conv2d(w.shape[1], C, 5, padding=2).to(dev())
    bn = pdt.SyncBatchNorm(C, momentum=momentum, process_group=group).to(dev())
    with torch.no_grad():
        conv.weight.copy_(w)
        conv.bias.copy_(b)
        bn.weight.copy_(gamma)
        bn.bias.copy_(beta)
        bn.running_mean.fill_(0.25)
        bn.running_var.fill_(2.0)
    ys = [_conv_y(nhwc(x), w, b) for x in xs]
    _queue_forward(group, "forward", ys, r, C)
    rec = _Recorder()
    mp.setattr(OF, "_C", rec)
    with torch.no_grad():
        out = ops.conv_bn_relu_pool(xs[r], conv, bn)
    mp.setattr(OF, "_C", _C)
    assert group.comm.calls == ["forward"] and group.comm.expected == []
    assert len(rec.ys) == 1 and torch.equal(rec.ys[0], ys[r])
    assert int(bn.num_batches_tracked) == 1
    return ys, out, bn


@pytest.mark.parametrize("ratio", RATIOS)
@pytest.mark.parametrize("ns,r", SHARDS)
@pytest.mark.parametrize("layer", [1, 2])
def test_layer_statistics_with_large_means(layer, ns, r, ratio, fake_dist):
    xs, w, b, gamma, beta, C = _layer_case(layer, ns, ratio, seed=3 + 10 * layer + sum(ns))
    ys, out, bn = _run_layer(xs, w, b, gamma, beta, C, r, 1.0, fake_dist)
    v = torch.cat([y.double().reshape(-1, C) for y in ys])
    # momentum 1: the running statistics are the group's own batch mean and (unbiased) variance
    mean, var, var_tol = _check_running(bn.running_mean, bn.running_var, 0.25, 2.0, 1.0, v, f"layer {layer}")
    _check_out(out, ys[r], mean, var, var_tol, gamma, beta, bn.eps)
    # a second run repeats the output and the running statistics bit for bit
    _, out2, bn2 = _run_layer(xs, w, b, gamma, beta, C, r, 1.0, fake_dist)
    assert torch.equal(out, out2)
    assert torch.equal(bn.running_mean, bn2.running_mean) and torch.equal(bn.running_var, bn2.running_var)


def test_layer_statistics_with_momentum(fake_dist):
    """momentum 0.1: the group's statistics enter the running statistics a tenth at a time."""
    ns, r = SHARDS[1]
    xs, w, b, gamma, beta, C = _layer_case(2, ns, 300, seed=41)
    ys, out, bn = _run_layer(xs, w, b, gamma, beta, C, r, 0.1, fake_dist)
    v = torch.cat([y.double().reshape(-1, C) for y in ys])
    mean, var, var_tol = _check_running(bn.running_mean, bn.running_var, 0.25, 2.0, 0.1, v, "layer 2")
    _check_out(out, ys[r], mean, var, var_tol, gamma, beta, bn.eps)


# ---- one training step of the ConvNet, then an eval forward -----------------------------------------------------------------------
STEP_RATIO = 300


def _convnet_step(ns, r, x, t, mp):
    xs, ts = list(x.split(list(ns))), list(t.split(list(ns)))
    group = _FakeGroup(len(ns))
    torch.manual_seed(5)
    net = pdt.SyncBatchNorm.convert_sync_batchnorm(pdt.models.ConvNet(), process_group=group).to(dev())
    _offset_biases(net, x, STEP_RATIO)
    # momentum 1: the running statistics are this batch's, so that the eval forward below depends on every digit of them
    net.layer1[1].momentum = net.layer2[1].momentum = 1.0
    twins = [_float64_twin(net) for _ in ns]
    for tw in twins:
        tw.layer1[1].momentum = tw.layer2[1].momentum = 1.0
    layers, logits_ref, losses = _convnet_oracle(twins, xs, ts)

    # the other ranks' conv outputs from the kernels: conv1 on their images, conv2 on their float64 layer-1 outputs
    c1, c2 = net.layer1[0], net.layer2[0]
    ys1 = [_conv_y(nhwc(xk), c1.weight, c1.bias) for xk in xs]
    h1 = [F.max_pool2d(F.relu(z.detach()), 2, 2).float() for z in layers[1]["zs"]]
    ys2 = [_conv_y(nhwc(h), c2.weight, c2.bias) for h in h1]
    _queue_forward(group, "layer1 forward", ys1, r, 16)
    _queue_forward(group, "layer2 forward", ys2, r, 32)
    others = lambda per: sum(p for k, p in enumerate(per) if k != r)  # noqa: E731
    for l in (2, 1):
        L = layers[l]
        xhat = [(y.detach() - L["mean"].detach().view(1, -1, 1, 1)) * L["invstd"].detach().view(1, -1, 1, 1) for y in L["ys"]]
        bwd = [torch.cat([z.grad.sum((0, 2, 3)), (z.grad * xh).sum((0, 2, 3))]) for z, xh in zip(L["zs"], xhat)]
        group.comm.expected.append((f"layer{l} backward", torch.float32, 2 * L["mean"].numel(), others(bwd), None))

    xr = xs[r].contiguous()
    assert not OF.fused_convnet_ok(xr, net)   # SyncBatchNorm takes the per-op kernels
    rec = _Recorder()
    mp.setattr(OF, "_C", rec)
    logits = net(xr)
    loss = pdt.nn.CrossEntropyLoss()(logits, ts[r])
    loss.backward()
    mp.setattr(OF, "_C", _C)
    assert group.comm.calls == ["layer1 forward", "layer2 forward", "layer2 backward", "layer1 backward"], group.comm.calls
    assert group.comm.expected == []
    assert len(rec.ys) == 2 and torch.equal(rec.ys[0], ys1[r])
    ys2[r] = rec.ys[1]   # this rank's conv2 output as the path computed it (its layer-1 output is the kernels')
    return dict(net=net, twins=twins, loss=loss, logits=logits, layers=layers, logits_ref=logits_ref, losses=losses,
                ys={1: ys1, 2: ys2}, xr=xr)


@pytest.mark.parametrize("ns,r", [SHARDS[0], SHARDS[3]])
def test_convnet_step_with_large_means_matches_float64(ns, r, fake_dist):
    gen = torch.Generator(device=dev()).manual_seed(9)
    x = torch.rand(sum(ns), 1, 28, 28, device=dev(), generator=gen)
    t = torch.randint(0, 10, (sum(ns),), device=dev(), generator=gen)
    s = _convnet_step(ns, r, x, t, fake_dist)
    net, layers = s["net"], s["layers"]

    # conv2 runs in TF32: loss, logits and gradients at test_syncbn_native.py's TF32 policy
    assert abs(s["loss"].item() - s["losses"][r].item()) < 2e-3, (s["loss"].item(), s["losses"][r].item())
    _norm_close(s["logits"].detach(), s["logits_ref"][r].detach(), "logits")
    for (name, p), (_, q) in zip(net.named_parameters(), s["twins"][r].named_parameters()):
        _norm_close(p.grad, q.grad, name, _grad_scale(name, layers, r))
    # the running statistics: float64 statistics of the conv outputs the group normalised
    for l, C in ((1, 16), (2, 32)):
        bn = getattr(net, f"layer{l}")[1]
        assert int(bn.num_batches_tracked) == 1
        v = torch.cat([y.double().reshape(-1, C) for y in s["ys"][l]])
        _check_running(bn.running_mean, bn.running_var, 0.0, 1.0, 1.0, v, f"layer {l}")

    # an eval forward with the updated running statistics against the float64 twin holding the oracle's
    ref = _float64_twin(net)
    with torch.no_grad():
        for l in (1, 2):
            getattr(ref, f"layer{l}")[1].running_mean.copy_(layers[l]["rm"])
            getattr(ref, f"layer{l}")[1].running_var.copy_(layers[l]["rv"])
    net.eval()
    ref.eval()
    with torch.no_grad():
        out, ref_out = net(s["xr"]), ref(s["xr"].double())
    # TF32 in conv2, and y ≈ r·spread in fp32 (ulp 2⁻²³·r of the spread) magnified by 1/spread in both layers
    err = (out.double() - ref_out).abs().max().item()
    assert err <= 1e-2 * ref_out.abs().max().item(), (err, ref_out.abs().max().item())

    # the whole step repeats bit for bit
    s2 = _convnet_step(ns, r, x, t, fake_dist)
    assert torch.equal(s["loss"], s2["loss"]) and torch.equal(s["logits"], s2["logits"])
    net2 = s2["net"]
    for (n1, p1), (_, p2) in zip(s["net"].named_parameters(), net2.named_parameters()):
        assert torch.equal(p1.grad, p2.grad), n1
    for (n1, b1), (_, b2) in zip(s["net"].named_buffers(), net2.named_buffers()):
        assert torch.equal(b1, b2), n1


# ---- two real ranks: DDP, one eager step and three replays of the graph-captured step --------------------------------------------
LR = 0.01


def _batch(rank, step, bs=100):
    g = torch.Generator().manual_seed(7000 + 100 * step + rank)
    return torch.rand(bs, 1, 28, 28, generator=g), torch.randint(0, 10, (bs,), generator=g)


def _group_batch(world, step):
    xs, ts = zip(*[_batch(k, step) for k in range(world)])
    return torch.cat(xs), torch.cat(ts)


def _ranks_step(rank, world):
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    dev_r = torch.device("cuda", rank)
    torch.manual_seed(0)
    model = pdt.SyncBatchNorm.convert_sync_batchnorm(pdt.models.ConvNet()).to(dev_r)
    _offset_biases(model, _group_batch(world, 0)[0].to(dev_r), STEP_RATIO)
    model.layer1[1].momentum = model.layer2[1].momentum = 1.0
    init = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    opt = pdt.optim.SGD(model.parameters(), LR)
    ddp = pdt.DistributedDataParallel(model, device_ids=[rank])
    crit = pdt.nn.CrossEntropyLoss()
    x, t = _batch(rank, 0)
    loss = crit(ddp(x.to(dev_r)), t.to(dev_r))
    opt.zero_grad()
    loss.backward()
    opt.step()
    x, t = _batch(rank, 1)
    step = GraphedTrainStep(ddp, crit, opt, (x.to(dev_r), t.to(dev_r)))   # its warm-up steps train on batch 1
    torch.cuda.synchronize(dev_r)
    warm = int(model.layer1[1].num_batches_tracked) - 1
    for s in (2, 3, 4):
        x, t = _batch(rank, s)
        step(x.pin_memory(), t.pin_memory())
    torch.cuda.synchronize(dev_r)
    return dict(init=init, warm=warm, state={k: v.detach().cpu().clone() for k, v in model.state_dict().items()})


@pytest.mark.multigpu
def test_ranks_graphed_steps_with_large_means_match_float64():
    """Two ranks on the NVLink backend: after one eager step, the graph-captured step's warm-up and three replays, every rank holds
    the parameters and running statistics of a float64 twin trained by SGD on the concatenated batches, and the ranks agree bit
    for bit."""
    world = 2
    res = run_ranks(_ranks_step, world, backend="nvlink")
    for k in res[0]["state"]:
        assert all(torch.equal(res[0]["state"][k], o["state"][k]) for o in res[1:]), k
    assert all(torch.equal(res[0]["init"][k], o["init"][k]) for o in res[1:] for k in res[0]["init"])
    warm = res[0]["warm"]
    assert warm >= 2 and int(res[0]["state"]["layer1.1.num_batches_tracked"]) == 1 + warm + 3

    ref = pdt.models.ConvNet(fused=False).to(dev())
    ref.load_state_dict(res[0]["init"])
    ref = ref.double()
    ref.layer1[1].momentum = ref.layer2[1].momentum = 1.0
    p0 = {n: p.detach().clone() for n, p in ref.named_parameters()}
    gsum = {n: 0.0 for n in p0}
    steps = [0] + [1] * warm + [2, 3, 4]
    for s in steps:
        x, t = _group_batch(world, s)
        ref.zero_grad()
        # DDP averages the ranks' mean losses: with equal shards, the mean loss of the concatenated batch
        F.cross_entropy(ref(x.to(dev()).double()), t.to(dev())).backward()
        with torch.no_grad():
            for n, p in ref.named_parameters():
                gsum[n] += p.grad.norm().item()
                p -= LR * p.grad
    state = res[0]["state"]
    for n, p in ref.named_parameters():
        # each step's gradient at the TF32 policy of the single-step tests, summed over the steps
        err = (state[n].double().to(dev()) - p.detach()).norm().item()
        tol = LR * (3e-2 * gsum[n] + len(steps) * 1e-4 * p.numel() ** 0.5)
        assert err <= tol, (n, err, tol, (p.detach() - p0[n]).norm().item())
    for n, b in ref.named_buffers():
        if n.endswith("num_batches_tracked"):
            continue
        # the last batch's statistics of the TF32 conv2 output; fp32 Σy²/n − mean² would be 2 % off the variance at r = 300
        got = state[n].double().to(dev())
        assert torch.allclose(got, b, atol=2e-3, rtol=1e-3), (n, ((got - b).abs() / b.abs()).max().item())
