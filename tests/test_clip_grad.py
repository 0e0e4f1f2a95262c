"""Gradient-norm clipping: pdt.nn.utils.clip_grad_norm_ against torch on the CPU (torch's path) and on the GPU (the native
norm and scale kernels), the clipping riders of the layer-1 backward kernel, GraphedTrainStep(max_grad_norm=...) and
train_mnist.py --clip-grad-norm."""
import math
import os
import subprocess
import sys

import pytest
import torch

import pytorch_distributed_train_b200 as pdt
from pytorch_distributed_train_b200.nn.utils import clip_grad_norm_

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NORMS = [2.0, math.inf]


def _params(shapes, seed, device="cpu", scale=1.0):
    g = torch.Generator().manual_seed(seed)
    ps = [torch.zeros(s, device=device, requires_grad=True) for s in shapes]
    for p in ps:
        p.grad = (torch.randn(p.shape, generator=g) * scale).to(device)
    return ps


def _clone(ps):
    out = []
    for p in ps:
        q = p.detach().clone().requires_grad_()
        q.grad = None if p.grad is None else p.grad.clone()
        out.append(q)
    return out


# =====================================================================================================================
# CPU: torch's path, bit for bit
# =====================================================================================================================
@pytest.mark.parametrize("norm_type", [2.0, math.inf, 1.0])
@pytest.mark.parametrize("max_norm", [0.5, 1e6])
def test_cpu_matches_torch_bit_for_bit(norm_type, max_norm):
    a = _params([(5, 3), (7,), (4, 4), (1,)], 0)
    a[2].grad = None   # a parameter without a gradient is skipped
    b = _clone(a)
    na = clip_grad_norm_(a, max_norm, norm_type)
    nb = torch.nn.utils.clip_grad_norm_(b, max_norm, norm_type)
    assert torch.equal(na, nb)
    for p, q in zip(a, b):
        assert (p.grad is None and q.grad is None) or torch.equal(p.grad, q.grad)


def test_cpu_empty_set_and_lone_tensor():
    assert torch.equal(clip_grad_norm_([], 1.0), torch.nn.utils.clip_grad_norm_([], 1.0))
    assert torch.equal(clip_grad_norm_([torch.zeros(3, requires_grad=True)], 1.0), torch.tensor(0.0))
    a = _params([(6, 2)], 1)[0]
    b = _clone([a])[0]
    assert torch.equal(clip_grad_norm_(a, 0.1), torch.nn.utils.clip_grad_norm_(b, 0.1))
    assert torch.equal(a.grad, b.grad)


@pytest.mark.parametrize("bad", [math.nan, math.inf])
def test_cpu_error_if_nonfinite_message(bad):
    a = _params([(4,), (3,)], 2)
    a[1].grad[0] = bad
    with pytest.raises(RuntimeError) as ours:
        clip_grad_norm_(a, 1.0, error_if_nonfinite=True)
    with pytest.raises(RuntimeError) as theirs:
        torch.nn.utils.clip_grad_norm_(_clone(a), 1.0, error_if_nonfinite=True)
    assert str(ours.value) == str(theirs.value)


def test_cli_rejects_non_positive_clip():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py"), "--clip-grad-norm", "0"],
                         capture_output=True, text=True, timeout=60, cwd=ROOT)
    assert out.returncode != 0 and "--clip-grad-norm must be positive" in out.stderr
    from pytorch_distributed_train_b200 import cli

    assert cli.build_parser().parse_args([]).clip_grad_norm is None


def _torch_ddp_clip(rank, world, port, steps, lr, max_norm):
    """torch DDP + gloo + torch.nn.utils.clip_grad_norm_ on train_mnist.py's data, model and seed."""
    import torch.distributed as td

    from pytorch_distributed_train_b200 import data as pdata

    td.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", world_size=world, rank=rank)
    try:
        torch.manual_seed(0)
        model = pdt.models.ConvNet()
        ddp = torch.nn.parallel.DistributedDataParallel(model)
        opt = torch.optim.SGD(ddp.parameters(), lr)
        crit = torch.nn.CrossEntropyLoss()
        ds = pdata.SyntheticMNIST(600, seed=0, num_classes=10, image_shape=(1, 28, 28))
        loader = torch.utils.data.DataLoader(ds, batch_size=100, shuffle=False,
                                             sampler=torch.utils.data.DistributedSampler(ds, num_replicas=world, rank=rank))
        norms = []
        for i, (x, y) in enumerate(loader):
            if i >= steps:
                break
            loss = crit(ddp(x), y)
            opt.zero_grad()
            loss.backward()
            norms.append(torch.nn.utils.clip_grad_norm_(ddp.parameters(), max_norm).item())
            opt.step()
        return {k: v.clone() for k, v in ddp.state_dict().items()}, norms
    finally:
        td.destroy_process_group()


def test_train_script_clip_matches_torch_ddp_gloo(tmp_path):
    from mp_helpers import free_port, run_ranks

    ck = str(tmp_path / "clip.pt")
    cmd = [sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "2", "--backend", "gloo", "--lr", "0.1", "--clip-grad-norm", "0.5",
           "--steps", "3", "--samples", "600", "--epochs", "1", "--log-interval", "3", "--checkpoint", ck]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=240, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "Epoch [1/1], Step [3/3]" in out.stdout
    ours = torch.load(ck, map_location="cpu", weights_only=False)["model"]
    ref, norms = run_ranks(_torch_ddp_clip, 2, free_port(), 3, 0.1, 0.5)[0]
    assert max(norms) > 0.5, norms   # clipping engaged
    assert list(ours) == list(ref)
    for k in ref:
        assert torch.allclose(ours[k].float(), ref[k].float(), atol=1e-5, rtol=1e-4), (k, (ours[k].float() - ref[k].float()).abs().max())


# =====================================================================================================================
# GPU
# =====================================================================================================================
def _dev():
    return torch.device("cuda", 0)


# more than 48 tensors (the fold spans two tables), with empty, tiny and large ones
SHAPES = [(0,), (1,), (3,), (1000000,)] + [(int(s),) for s in torch.randint(1, 5000, (56,), generator=torch.Generator().manual_seed(3))]


def _f64_norm(grads, norm_type):
    flat = torch.cat([g.double().reshape(-1) for g in grads])
    return flat.abs().max().item() if norm_type == math.inf else flat.norm().item()


@pytest.mark.gpu
@pytest.mark.parametrize("norm_type", NORMS)
@pytest.mark.parametrize("where", ["below", "above"])
def test_kernel_matches_float64_and_torch(norm_type, where):
    from pytorch_distributed_train_b200 import _C

    # torch refuses the inf-norm of an empty tensor (and so does ours, through torch's path)
    a = _params(SHAPES if norm_type == 2.0 else SHAPES[1:], 4, _dev())
    b = _clone(a)
    orig = [p.grad.clone() for p in a]
    ref = _f64_norm(orig, norm_type)
    max_norm = ref * (0.3 if where == "below" else 3.0)
    c0 = _C.kernel_launch_count()
    na = clip_grad_norm_(a, max_norm, norm_type)
    assert _C.kernel_launch_count() - c0 == 4, "two tables: two norm and two scale launches"
    nb = torch.nn.utils.clip_grad_norm_(b, max_norm, norm_type)
    torch.cuda.synchronize()
    assert na.dtype == torch.float32 and na.device == _dev() and na.dim() == 0
    if norm_type == math.inf:
        assert na.item() == nb.item() == ref
    else:
        assert abs(na.item() - ref) <= 1e-5 * ref and abs(na.item() - nb.item()) <= 1e-5 * ref
    for p, q, g in zip(a, b, orig):
        if where == "above":   # coefficient 1: the gradients stay as they were, as torch leaves them
            assert torch.equal(p.grad, q.grad) and torch.equal(p.grad, g)
        else:
            assert torch.allclose(p.grad, q.grad, rtol=1e-5, atol=0), (p.grad - q.grad).abs().max().item()
            if p.numel():
                exp = g.double() * (max_norm / (ref + 1e-6))
                assert torch.allclose(p.grad.double(), exp, rtol=1e-5, atol=0)


@pytest.mark.gpu
@pytest.mark.parametrize("norm_type", NORMS)
def test_norm_is_bit_reproducible(norm_type):
    from pytorch_distributed_train_b200 import ops

    a = _params(SHAPES, 5, _dev())
    grads = [p.grad for p in a]
    n1 = ops.grad_norm_clip(grads, 1.0, norm_type, scale=False).clone()
    n2 = ops.grad_norm_clip(grads, 1.0, norm_type, scale=False).clone()
    assert torch.equal(n1, n2)


@pytest.mark.gpu
def test_inf_norm_of_an_empty_gradient_raises_as_torch_does():
    a = _params([(0,), (3,)], 9, _dev())
    with pytest.raises(RuntimeError) as ours:
        clip_grad_norm_(a, 1.0, math.inf)
    with pytest.raises(RuntimeError) as theirs:
        torch.nn.utils.clip_grad_norm_(_clone(a), 1.0, math.inf)
    assert str(ours.value) == str(theirs.value)


@pytest.mark.gpu
@pytest.mark.parametrize("norm_type", NORMS)
@pytest.mark.parametrize("bad", [math.nan, math.inf])
def test_nonfinite_gradients_follow_torch(norm_type, bad):
    a = _params([(100,), (7, 3), (1,)], 6, _dev())
    a[1].grad[2, 1] = bad
    b = _clone(a)
    orig = [p.grad.clone() for p in a]
    na = clip_grad_norm_(a, 1.0, norm_type)
    nb = torch.nn.utils.clip_grad_norm_(b, 1.0, norm_type)
    torch.testing.assert_close(na, nb, rtol=0, atol=0, equal_nan=True)
    for p, q in zip(a, b):
        torch.testing.assert_close(p.grad, q.grad, rtol=0, atol=0, equal_nan=True)
    c = _params([(100,), (7, 3), (1,)], 6, _dev())
    c[1].grad[2, 1] = bad
    with pytest.raises(RuntimeError, match="is non-finite, so it cannot be clipped"):
        clip_grad_norm_(c, 1.0, norm_type, error_if_nonfinite=True)
    for p, g in zip(c, orig):   # raised before anything was scaled
        torch.testing.assert_close(p.grad, g, rtol=0, atol=0, equal_nan=True)


@pytest.mark.gpu
def test_captured_clip_tracks_eager_on_replay():
    a = _params([(300,), (17, 5), (1,), (4000,)], 7, _dev())
    grads = [p.grad for p in a]
    clip_grad_norm_(a, 1.0)   # the reduction scratch exists before the capture
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        norm = clip_grad_norm_(a, 1.0)
    gen = torch.Generator().manual_seed(8)
    for r in range(5):
        new = [torch.randn(g.shape, generator=gen).to(_dev()) * (0.01 if r % 2 else 1.0) for g in grads]
        for g, v in zip(grads, new):
            g.copy_(v)
        graph.replay()
        b = [torch.zeros_like(g, requires_grad=True) for g in grads]
        for q, v in zip(b, new):
            q.grad = v.clone()
        nb = torch.nn.utils.clip_grad_norm_(b, 1.0)
        torch.cuda.synchronize()
        assert abs(norm.item() - nb.item()) <= 1e-5 * nb.item()
        for g, q in zip(grads, b):
            assert torch.allclose(g, q.grad, rtol=1e-5, atol=0)


def _batch(s):
    g = torch.Generator(device=_dev()).manual_seed(s)
    return torch.rand(100, 1, 28, 28, device=_dev(), generator=g), torch.randint(0, 10, (100,), device=_dev(), generator=g)


def _riding_pair(kind):
    torch.manual_seed(4)
    a = pdt.models.ConvNet(fused=True).to(_dev())
    b = pdt.models.ConvNet(fused=True).to(_dev())
    b.load_state_dict(a.state_dict())
    if kind == "sgd":
        make = lambda m: pdt.optim.SGD(m.parameters(), 0.05, momentum=0.9)   # noqa: E731
    else:
        make = lambda m: pdt.optim.AdamW(m.parameters(), 1e-3, weight_decay=1e-2)   # noqa: E731
    return a, b, make(a), make(b)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sgd", "adamw"])
def test_clipping_rider_follows_eager_clip_and_step(kind):
    """The clipping rider (ClipRider) against an eager loop: backward, clip_grad_norm_, the multi-tensor optimizer kernel."""
    from pytorch_distributed_train_b200 import _C
    from pytorch_distributed_train_b200.ops import functional as OF

    a, b, oa, ob = _riding_pair(kind)
    crit = pdt.nn.CrossEntropyLoss()
    max_norm = 0.05
    # The two convolution biases feed a BatchNorm: their gradient is rounding noise.  The two paths fold the norm in different
    # orders, so the coefficients may differ in the last bit; after one update that noise differs, and Adam scales it up to
    # full-size steps.  With AdamW the biases are left out (as in test_adam.py's graphed step).
    skip = ("layer1.0.bias", "layer2.0.bias") if kind == "adamw" else ()
    norm_out = torch.zeros((), device=_dev())
    assert oa.ride_on_backward(a, clip=(max_norm, 2.0, norm_out))
    try:
        for s in range(4):
            x, t = _batch(s)
            before = _C.kernel_launch_count()
            oa.zero_grad()
            la = crit(a(x), t)
            with OF.sgd_rider_enabled():
                la.backward()
            assert oa._rode
            oa.step()
            riding = _C.kernel_launch_count() - before
            before = _C.kernel_launch_count()
            ob.zero_grad()
            crit(b(x), t).backward()
            nb = clip_grad_norm_(b.parameters(), max_norm)
            ob.step()
            eager = _C.kernel_launch_count() - before
            assert riding < eager, (riding, eager)
            torch.cuda.synchronize()
            assert nb.item() > max_norm, "clipping must engage"
            assert abs(norm_out.item() - nb.item()) <= 1e-4 * nb.item(), (norm_out.item(), nb.item())
            for (n1, p1), p2 in zip(a.named_parameters(), b.parameters()):
                if n1 in skip:
                    continue
                assert torch.allclose(p1, p2, atol=1e-6, rtol=1e-5), (s, n1, (p1 - p2).abs().max().item())
                assert torch.allclose(p1.grad, p2.grad, atol=1e-7, rtol=1e-4), (s, n1, (p1.grad - p2.grad).abs().max().item())
        for (n1, p1), p2 in zip(a.named_parameters(), b.parameters()):
            s1, s2 = oa.state[p1], ob.state[p2]
            for k in s1:
                if n1 in skip and k != "step":
                    continue
                if k == "step":
                    assert s1[k].item() == s2[k].item() == 4.0
                else:
                    assert torch.allclose(s1[k], s2[k], atol=1e-7, rtol=1e-5), k
    finally:
        oa.stop_riding()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sgd", "adamw"])
def test_clipping_rider_far_above_the_norm_equals_plain_rider(kind):
    from pytorch_distributed_train_b200.ops import functional as OF

    a, b, oa, ob = _riding_pair(kind)
    crit = pdt.nn.CrossEntropyLoss()
    norm_out = torch.zeros((), device=_dev())
    for s in range(3):
        x, t = _batch(10 + s)
        for model, opt, clip in ((a, oa, (1e9, 2.0, norm_out)), (b, ob, None)):
            assert opt.ride_on_backward(model, clip=clip)
            opt.zero_grad()
            loss = crit(model(x), t)
            with OF.sgd_rider_enabled():
                loss.backward()
            assert opt._rode
            opt.step()
            opt.stop_riding()
        for p1, p2 in zip(a.parameters(), b.parameters()):
            assert torch.equal(p1, p2)
            assert torch.equal(p1.grad, p2.grad)
    assert 0 < norm_out.item() < 1e9


def _graphed_vs_torch(opt_kind, two_groups):
    from mp_helpers import free_port

    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    torch.cuda.set_device(0)
    pdt.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{free_port()}", world_size=1, rank=0)
    try:
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(_dev())
        ref = pdt.models.ConvNet().to(_dev())
        ref.load_state_dict(model.state_dict())
        ps = list(model.parameters())
        groups = [{"params": ps[:6]}, {"params": ps[6:]}] if two_groups else ps
        if opt_kind == "sgd":
            opt, ropt = pdt.optim.SGD(groups, 0.05), torch.optim.SGD(ref.parameters(), 0.05)
        else:
            opt, ropt = pdt.optim.AdamW(groups, 1e-3), torch.optim.AdamW(ref.parameters(), 1e-3, foreach=False)
        ddp = pdt.DistributedDataParallel(model, device_ids=[0])
        crit = pdt.nn.CrossEntropyLoss()
        g = torch.Generator(device=_dev()).manual_seed(9)
        xs = torch.rand(4, 100, 1, 28, 28, device=_dev(), generator=g)
        ts = torch.randint(0, 10, (4, 100), device=_dev(), generator=g)
        max_norm = 0.5
        step = GraphedTrainStep(ddp, crit, opt, (xs[0], ts[0]), warmup=3, max_grad_norm=max_norm)
        kernels = step.kernels_per_replay
        warm = 3

        def ref_step(x, t):
            ropt.zero_grad()
            crit(ref(x), t).backward()
            n = torch.nn.utils.clip_grad_norm_(ref.parameters(), max_norm)
            ropt.step()
            return n

        for _ in range(warm):
            ref_step(xs[0], ts[0])
        norms = []
        for i in range(20):
            step(xs[i % 4], ts[i % 4], inputs_ready=True)
            norms.append((step.grad_norm.item(), ref_step(xs[i % 4], ts[i % 4]).item()))
        torch.cuda.synchronize()
        keep = [(p, q) for (n, p), q in zip(model.named_parameters(), ref.parameters()) if n not in ("layer1.0.bias", "layer2.0.bias")]
        ours_flat = torch.cat([p.detach().reshape(-1) for p, _ in keep])
        ref_flat = torch.cat([q.detach().reshape(-1) for _, q in keep])
        err = (ours_flat - ref_flat).abs().max().item() / ref_flat.abs().max().item()
        return kernels, err, norms
    finally:
        pdt.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("opt_kind", ["sgd", "adamw"])
def test_graphed_step_with_clipping_is_three_launches_and_follows_torch(opt_kind):
    kernels, err, norms = _graphed_vs_torch(opt_kind, two_groups=False)
    assert kernels == 3, kernels
    assert err < 2e-2, err
    assert all(r > 0.5 for _, r in norms), "clipping must engage"
    # the first replay's norm comes from the same parameters up to the warm-up steps' rounding
    assert abs(norms[0][0] - norms[0][1]) <= 1e-3 * norms[0][1], norms[0]
    assert all(abs(o - r) <= 2e-2 * r for o, r in norms), norms


@pytest.mark.gpu
def test_graphed_step_clips_between_backward_and_step_when_not_riding():
    """Two parameter groups do not ride: the native clip (norm + scale) runs inside the graph before the optimizer's own
    launches (one per group)."""
    kernels, err, norms = _graphed_vs_torch("sgd", two_groups=True)
    assert kernels == 3 + 2 + 2, kernels
    assert err < 2e-2, err
    assert all(abs(o - r) <= 2e-2 * r for o, r in norms), norms


def _graphed_clip_n2(rank, world, port):
    import torch.distributed as td

    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    dev = torch.device("cuda", rank)
    g = torch.Generator().manual_seed(100 + rank)
    xs, ts = torch.rand(4, 100, 1, 28, 28, generator=g), torch.randint(0, 10, (4, 100), generator=g)
    torch.manual_seed(0)
    model = pdt.models.ConvNet().to(dev)
    opt = pdt.optim.AdamW(model.parameters(), 1e-3)
    ddp = pdt.DistributedDataParallel(model, device_ids=[rank])
    crit = pdt.nn.CrossEntropyLoss()
    step = GraphedTrainStep(ddp, crit, opt, (xs[0].to(dev), ts[0].to(dev)), warmup=3, max_grad_norm=0.5)
    for i in range(10):
        step(xs[i % 4].pin_memory(), ts[i % 4].pin_memory())
    torch.cuda.synchronize()
    ours = torch.cat([p.detach().reshape(-1) for p in ddp.parameters()]).cpu()
    warm = int(next(iter(opt.state.values()))["step"].item()) - 10

    td.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", world_size=world, rank=rank)
    try:
        torch.manual_seed(0)
        ref = pdt.models.ConvNet().to(dev)
        rddp = torch.nn.parallel.DistributedDataParallel(ref, device_ids=[rank])
        ropt = torch.optim.AdamW(rddp.parameters(), 1e-3, foreach=False)
        for i in [0] * warm + [i % 4 for i in range(10)]:
            ropt.zero_grad()
            torch.nn.functional.cross_entropy(rddp(xs[i].to(dev)), ts[i].to(dev)).backward()
            torch.nn.utils.clip_grad_norm_(rddp.parameters(), 0.5)
            ropt.step()
        theirs = torch.cat([p.detach().reshape(-1) for p in rddp.parameters()]).cpu()
    finally:
        td.destroy_process_group()
    return ours, theirs, step.kernels_per_replay


@pytest.mark.gpu
@pytest.mark.multigpu
def test_graphed_step_with_clipping_at_two_gpus_follows_torch_ddp():
    from mp_helpers import free_port, run_ranks

    res = run_ranks(_graphed_clip_n2, 2, free_port(), backend="nccl")
    assert torch.equal(res[0][0], res[1][0]), "ranks must stay bit-identical"
    for ours, theirs, _ in res:
        assert (ours - theirs).abs().max().item() < 2e-2 * theirs.abs().max().item()
