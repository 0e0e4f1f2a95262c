"""pdt.optim.Adam / AdamW: torch's semantics on the CPU (reference math), the multi-tensor sm_90a kernel, the rider of the
layer-1 backward kernel and the whole-step CUDA graph on the GPU."""
import copy
import os
import subprocess
import sys

import pytest
import torch

import pytorch_distributed_train_b200 as pdt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAIRS = [(pdt.optim.Adam, torch.optim.Adam), (pdt.optim.AdamW, torch.optim.AdamW)]


def _two_groups(seed, device="cpu"):
    g = torch.Generator().manual_seed(seed)
    a = [torch.randn(5, 3, generator=g), torch.randn(7, generator=g)]
    b = [torch.randn(4, 4, generator=g)]
    return [[t.to(device).requires_grad_() for t in a], [t.to(device).requires_grad_() for t in b]]


def _clone(groups):
    return [[t.detach().clone().requires_grad_() for t in grp] for grp in groups]


def _set_grads(groups_list, seed):
    g = torch.Generator().manual_seed(seed)
    for grp in zip(*groups_list):
        for ts in zip(*grp):
            v = torch.randn(ts[0].shape, generator=g).to(ts[0].device)
            for t in ts:
                t.grad = v.clone()


@pytest.mark.parametrize("ours,theirs", PAIRS)
@pytest.mark.parametrize("kw", [dict(), dict(weight_decay=0.1), dict(maximize=True, weight_decay=1e-2), dict(amsgrad=True),
                                dict(amsgrad=True, maximize=True, weight_decay=0.05, betas=(0.8, 0.99), eps=1e-6)])
def test_matches_torch_over_five_steps_with_two_groups(ours, theirs, kw):
    ga = _two_groups(0)
    gb = _clone(ga)
    a = ours([{"params": ga[0]}, {"params": ga[1], "lr": 3e-2}], lr=1e-2, **kw)
    b = theirs([{"params": gb[0]}, {"params": gb[1], "lr": 3e-2}], lr=1e-2, foreach=False, **kw)
    for s in range(5):
        _set_grads([ga, gb], s)
        a.step()
        b.step()
    for pa, pb in zip(sum(ga, []), sum(gb, [])):
        assert torch.allclose(pa, pb, rtol=1e-6, atol=1e-7), (pa - pb).abs().max()
        sa, sb = a.state[pa], b.state[pb]
        assert set(sa) == set(sb)
        for k in sa:
            assert torch.allclose(sa[k].float(), sb[k].float(), rtol=1e-6, atol=1e-7), k


@pytest.mark.parametrize("ours,theirs", PAIRS)
@pytest.mark.parametrize("kw", [dict(lr=-1.0), dict(eps=-1e-8), dict(betas=(1.0, 0.999)), dict(betas=(0.9, -0.1)),
                                dict(weight_decay=-1e-3), dict(betas=(0.9, torch.tensor(0.999))),
                                dict(lr=torch.tensor([1e-3, 1e-3]))])
def test_constructor_errors_match_torch(ours, theirs, kw):
    p = [torch.zeros(3, requires_grad=True)]
    with pytest.raises(ValueError) as want:
        theirs(p, **kw)
    with pytest.raises(ValueError) as got:
        ours(p, **kw)
    assert str(got.value) == str(want.value)


def test_defaults_match_torch():
    p = [torch.zeros(3, requires_grad=True)]
    for ours, theirs in PAIRS:
        da, db = ours(p).defaults, theirs(p).defaults
        assert da == db, (da, db)
    assert pdt.optim.AdamW(p).defaults["weight_decay"] == 1e-2


@pytest.mark.parametrize("ours,theirs", PAIRS)
@pytest.mark.parametrize("direction", ["pdt_to_torch", "torch_to_pdt"])
def test_state_dict_moves_between_pdt_and_torch(ours, theirs, direction):
    ga = _two_groups(1)
    gb = _clone(ga)
    src_cls, dst_cls = (ours, theirs) if direction == "pdt_to_torch" else (theirs, ours)
    src = src_cls([{"params": ga[0]}, {"params": ga[1]}], lr=1e-2, weight_decay=1e-2)
    for s in range(2):
        _set_grads([ga], 10 + s)
        src.step()
    with torch.no_grad():
        for pa, pb in zip(sum(ga, []), sum(gb, [])):
            pb.copy_(pa)
    dst = dst_cls([{"params": gb[0]}, {"params": gb[1]}], lr=5.0)
    dst.load_state_dict(copy.deepcopy(src.state_dict()))   # as through a file: no tensor shared with the source
    assert dst.param_groups[0]["lr"] == 1e-2
    for p in sum(gb, []):
        assert dst.state[p]["step"].item() == 2.0
    for s in range(3):
        _set_grads([ga, gb], 20 + s)
        src.step()
        dst.step()
    for pa, pb in zip(sum(ga, []), sum(gb, [])):
        assert torch.allclose(pa, pb, rtol=1e-6, atol=1e-7)
        assert torch.allclose(src.state[pa]["exp_avg_sq"], dst.state[pb]["exp_avg_sq"], rtol=1e-6, atol=1e-9)


def test_train_script_adamw_checkpoint_and_resume(tmp_path):
    ck = str(tmp_path / "adamw.pt")
    base = [sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "2", "--backend", "gloo", "--optimizer", "adamw", "--lr", "1e-3",
            "--steps", "3", "--samples", "600", "--log-interval", "3"]
    a = subprocess.run(base + ["--epochs", "1", "--checkpoint", ck], capture_output=True, text=True, timeout=240, cwd=ROOT)
    assert a.returncode == 0 and os.path.exists(ck), a.stderr[-2000:]
    saved = torch.load(ck, map_location="cpu", weights_only=False)["optimizer"]
    assert saved["param_groups"][0]["decoupled_weight_decay"] is True and saved["param_groups"][0]["weight_decay"] == 1e-2
    assert all(float(st["step"]) == 3.0 and "exp_avg_sq" in st for st in saved["state"].values())
    b = subprocess.run(base + ["--epochs", "2", "--resume", ck], capture_output=True, text=True, timeout=240, cwd=ROOT)
    assert b.returncode == 0, b.stderr[-2000:]
    assert "Resumed from" in b.stdout and "Epoch [2/2], Step [3/3]" in b.stdout and "Epoch [1/2]" not in b.stdout


def test_cli_rejects_momentum_with_adam():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py"), "--optimizer", "adam", "--momentum", "0.9"],
                         capture_output=True, text=True, timeout=60, cwd=ROOT)
    assert out.returncode != 0 and "--momentum applies to SGD only" in out.stderr
    from pytorch_distributed_train_b200 import cli

    a = cli.build_parser().parse_args([])
    assert a.optimizer == "sgd" and isinstance(cli.make_optimizer(a, [torch.zeros(1, requires_grad=True)]), pdt.optim.SGD)


# =====================================================================================================================
# GPU
# =====================================================================================================================
def _dev():
    return torch.device("cuda", 0)


def _adam_f64(p, m, v, step, grads, lr, beta1, beta2, eps, wd, decoupled, maximize):
    """The same formula in float64 (the oracle of the kernel's arithmetic)."""
    for g in grads:
        g = -g if maximize else g
        step += 1
        if wd:
            if decoupled:
                p = p * (1 - lr * wd)
            else:
                g = g + wd * p
        m = m + (1 - beta1) * (g - m)
        v = beta2 * v + (1 - beta2) * g * g
        p = p - (lr / (1 - beta1 ** step)) * m / (v.sqrt() / (1 - beta2 ** step) ** 0.5 + eps)
    return p, m, v


CONVNET_SIZES = [(16, 1, 5, 5), (16,), (16,), (16,), (32, 16, 5, 5), (32,), (32,), (32,), (10, 1568), (10,)]


@pytest.mark.gpu
@pytest.mark.parametrize("ours,theirs", PAIRS)
@pytest.mark.parametrize("kw", [dict(weight_decay=0.0), dict(weight_decay=1e-2), dict(weight_decay=1e-2, maximize=True)])
def test_kernel_matches_torch_and_float64_over_ten_steps(ours, theirs, kw):
    from pytorch_distributed_train_b200 import _C

    torch.manual_seed(5)
    shapes = CONVNET_SIZES + [(1,), (3,), (100003,)]
    pa = [torch.randn(s, device=_dev()).requires_grad_() for s in shapes]
    pb = [p.detach().clone().requires_grad_() for p in pa]
    init = [p.detach().double() for p in pa]
    a = ours(pa, lr=1e-2, **kw)
    b = theirs(pb, lr=1e-2, foreach=False, **kw)
    grads = [[torch.randn(s, device=_dev()) * 10 ** (i % 3 - 1) for s in shapes] for i in range(10)]
    launches = 0
    for gs in grads:
        for p, q, g in zip(pa, pb, gs):
            p.grad, q.grad = g.clone(), g.clone()
        c0 = _C.kernel_launch_count()
        a.step()
        launches += _C.kernel_launch_count() - c0
        b.step()
    assert launches == 10, "one multi-tensor launch per step"
    wd, decoupled = kw["weight_decay"], ours is pdt.optim.AdamW
    for i, (p, q) in enumerate(zip(pa, pb)):
        sa, sb = a.state[p], b.state[q]
        assert sa["step"].is_cuda and sa["step"].dtype == torch.float32 and sa["step"].item() == 10.0 == sb["step"].item()
        for x, y in ((p, q), (sa["exp_avg"], sb["exp_avg"]), (sa["exp_avg_sq"], sb["exp_avg_sq"])):
            assert torch.allclose(x, y, rtol=1e-5, atol=1e-7), (i, (x - y).abs().max().item())
        ref = _adam_f64(init[i], torch.zeros(shapes[i], dtype=torch.float64, device=_dev()), torch.zeros(shapes[i], dtype=torch.float64,
                        device=_dev()), 0, [gs[i].double() for gs in grads], 1e-2, 0.9, 0.999, 1e-8, wd, decoupled, kw.get("maximize", False))
        # against float64 the tolerance is relative to the largest magnitude the value was formed from: fp32 rounding of the
        # initial parameter, or of the largest gradient inside exp_avg, stays in an element that later passes near zero
        g_max = torch.stack([gs[i].abs() for gs in grads]).amax(0).double()
        for name, x, y, scale in (("p", p, ref[0], init[i].abs()), ("exp_avg", sa["exp_avg"], ref[1], g_max),
                                  ("exp_avg_sq", sa["exp_avg_sq"], ref[2], ref[2].abs())):
            err = (x.double() - y).abs()
            assert bool((err <= 1e-5 * torch.maximum(y.abs(), scale) + 1e-7).all()), (i, name, err.max().item())


@pytest.mark.gpu
def test_captured_step_advances_the_bias_corrections_on_replay():
    """One adam_step in a CUDA graph, replayed 20 times with the learning rate changed through sync_lr after 10: the same as 20 eager
    torch steps on that schedule — the step count (and with it the bias corrections) advances on every replay."""
    from pytorch_distributed_train_b200 import ops

    torch.manual_seed(6)
    shapes = [(300,), (17, 5), (1,)]
    pa = [torch.randn(s, device=_dev()).requires_grad_() for s in shapes]
    pb = [p.detach().clone().requires_grad_() for p in pa]
    for p, q in zip(pa, pb):
        p.grad = torch.randn_like(p)
        q.grad = p.grad.clone()
    a = pdt.optim.AdamW(pa, lr=1e-2, capturable=True)
    b = torch.optim.AdamW(pb, lr=1e-2, foreach=False)
    # everything a captured step reads must exist before the capture: the state, the learning-rate scalar, the kernel's scratch
    for p in pa:
        a._state(p, False)
    a._lr_tensor(0, a.param_groups[0], _dev())
    z = torch.zeros(4, device=_dev())
    ops.adam_step([z.clone()], [z.clone()], [z.clone()], [z.clone()], [torch.zeros((), device=_dev())], lr=0.0)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        a.step()
    assert all(a.state[p]["step"].item() == 0.0 for p in pa), "capturing must not run the step"
    for r in range(20):
        if r == 10:
            a.param_groups[0]["lr"] = b.param_groups[0]["lr"] = 3e-3
            a.sync_lr()
        graph.replay()
        b.step()
    torch.cuda.synchronize()
    for p, q in zip(pa, pb):
        assert a.state[p]["step"].item() == 20.0
        assert torch.allclose(p, q, rtol=1e-5, atol=1e-7), (p - q).abs().max().item()
        assert torch.allclose(a.state[p]["exp_avg"], b.state[q]["exp_avg"], rtol=1e-5, atol=1e-7)
        assert torch.allclose(a.state[p]["exp_avg_sq"], b.state[q]["exp_avg_sq"], rtol=1e-5, atol=1e-7)


@pytest.mark.gpu
@pytest.mark.parametrize("cls", [pdt.optim.Adam, pdt.optim.AdamW])
def test_adam_rider_rides_on_the_last_backward_kernel(cls):
    """Adam.ride_on_backward: the layer-1 backward kernel applies the update of all ten parameters (fused_convnet.cu: AdamRider);
    parameters and state must follow the separate multi-tensor Adam kernel."""
    from pytorch_distributed_train_b200 import _C
    from pytorch_distributed_train_b200.ops import functional as OF

    torch.manual_seed(4)
    a = pdt.models.ConvNet(fused=True).to(_dev())
    b = pdt.models.ConvNet(fused=True).to(_dev())
    b.load_state_dict(a.state_dict())
    oa = cls(a.parameters(), 1e-3, weight_decay=1e-2)
    ob = cls(b.parameters(), 1e-3, weight_decay=1e-2)
    crit = pdt.nn.CrossEntropyLoss()
    assert oa.ride_on_backward(a) and OF._sgd_rider.owner is oa
    try:
        for s in range(4):
            x = torch.rand(100, 1, 28, 28, device=_dev(), generator=torch.Generator(device=_dev()).manual_seed(s))
            t = torch.randint(0, 10, (100,), device=_dev(), generator=torch.Generator(device=_dev()).manual_seed(50 + s))
            before = _C.kernel_launch_count()
            oa.zero_grad()
            la = crit(a(x), t)
            if s == 0:   # outside the engine's context an armed optimizer must not touch the parameters
                la.backward()
                assert not oa._rode
                oa.zero_grad()
                before = _C.kernel_launch_count()
                la = crit(a(x), t)
            with OF.sgd_rider_enabled():
                la.backward()
            assert oa._rode, "the backward kernel should have applied the update"
            oa.step()
            riding = _C.kernel_launch_count() - before
            before = _C.kernel_launch_count()
            ob.zero_grad()
            crit(b(x), t).backward()
            ob.step()
            separate = _C.kernel_launch_count() - before
            assert riding < separate, (riding, separate)
            for (n1, p1), (_, p2) in zip(a.named_parameters(), b.named_parameters()):
                assert torch.allclose(p1, p2, atol=1e-6, rtol=1e-5), (s, n1, (p1 - p2).abs().max().item())
        for p1, p2 in zip(a.parameters(), b.parameters()):
            s1, s2 = oa.state[p1], ob.state[p2]
            assert s1["step"].item() == s2["step"].item() == 4.0
            assert torch.allclose(s1["exp_avg"], s2["exp_avg"], atol=1e-7, rtol=1e-5)
            assert torch.allclose(s1["exp_avg_sq"], s2["exp_avg_sq"], atol=1e-9, rtol=1e-5)
    finally:
        oa.stop_riding()


@pytest.mark.gpu
def test_graphed_step_with_adamw_is_three_launches_and_follows_torch():
    """engine.GraphedTrainStep with pdt.optim.AdamW on one GPU: the update rides on the last backward kernel (3 launches per
    replay), and 20 replays follow an eager loop with torch.optim.AdamW within bench.py's verification tolerance."""
    from mp_helpers import free_port

    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    torch.cuda.set_device(0)
    pdt.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{free_port()}", world_size=1, rank=0)
    try:
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(_dev())
        ref = pdt.models.ConvNet().to(_dev())
        ref.load_state_dict(model.state_dict())
        opt = pdt.optim.AdamW(model.parameters(), 1e-3)
        ropt = torch.optim.AdamW(ref.parameters(), 1e-3, foreach=False)
        ddp = pdt.DistributedDataParallel(model, device_ids=[0])
        crit = pdt.nn.CrossEntropyLoss()
        g = torch.Generator(device=_dev()).manual_seed(9)
        xs = torch.rand(4, 100, 1, 28, 28, device=_dev(), generator=g)
        ts = torch.randint(0, 10, (4, 100), device=_dev(), generator=g)
        step = GraphedTrainStep(ddp, crit, opt, (xs[0], ts[0]), warmup=3)
        assert step.kernels_per_replay == 3, step.kernels_per_replay
        # the engine's eager warm-up steps trained the model on the example batch: the reference loop takes them too
        warm = int(next(iter(opt.state.values()))["step"].item())
        assert warm >= 3
        for _ in range(warm):
            ropt.zero_grad()
            crit(ref(xs[0]), ts[0]).backward()
            ropt.step()
        for i in range(20):
            step(xs[i % 4], ts[i % 4], inputs_ready=True)
            ropt.zero_grad()
            crit(ref(xs[i % 4]), ts[i % 4]).backward()
            ropt.step()
        with torch.no_grad():
            ref_loss = crit(ref(xs[3]), ts[3])
        torch.cuda.synchronize()
        assert all(st["step"].item() == warm + 20 for st in opt.state.values())
        # bench.py's verification metric (max |ours − reference| / max |reference| over the flat vector, tolerance 2e-2), here on
        # the parameters.  The two convolution biases feed a BatchNorm: their gradient is rounding noise, which Adam scales up to
        # full-size steps, so they are left out.
        keep = [(p, q) for (n, p), q in zip(model.named_parameters(), ref.parameters()) if n not in ("layer1.0.bias", "layer2.0.bias")]
        ours_flat = torch.cat([p.detach().reshape(-1) for p, _ in keep])
        ref_flat = torch.cat([q.detach().reshape(-1) for _, q in keep])
        err = (ours_flat - ref_flat).abs().max().item() / ref_flat.abs().max().item()
        assert err < 2e-2, err
        # both models evaluated on the last batch after the last update (the graphed model through its eager path)
        with torch.no_grad():
            ours_loss = crit(model(xs[3]), ts[3]).item()
        assert abs(ours_loss - ref_loss.item()) < 2e-2 * ref_loss.item(), (ours_loss, ref_loss.item())
    finally:
        pdt.destroy_process_group()
