"""pdt.optim.Adam / AdamW with amsgrad=True on the native paths: the multi-tensor kernel (amsgrad_multi_kernel), the AMSGrad riders
of the layer-1 backward kernel, a captured step, GraphedTrainStep, state_dict exchange with torch and train_mnist.py --amsgrad.
On the CPU, amsgrad keeps torch's single-tensor arithmetic (test_adam.py)."""
import copy
import os
import subprocess
import sys

import pytest
import torch

import pytorch_distributed_train_b200 as pdt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAIRS = [(pdt.optim.Adam, torch.optim.Adam), (pdt.optim.AdamW, torch.optim.AdamW)]
CONVNET_SIZES = [(16, 1, 5, 5), (16,), (16,), (16,), (32, 16, 5, 5), (32,), (32,), (32,), (10, 1568), (10,)]
# the ConvNet's biases of the two convolutions feed a BatchNorm: their gradient is rounding noise, which Adam scales up to full-size
# steps, so comparisons of two different gradient paths leave them out
NOISE = ("layer1.0.bias", "layer2.0.bias")


# =====================================================================================================================
# CPU
# =====================================================================================================================
def test_cli_amsgrad_reaches_the_optimizer_and_sgd_refuses_it():
    from pytorch_distributed_train_b200 import cli

    p = [torch.zeros(1, requires_grad=True)]
    for name, cls in (("adam", pdt.optim.Adam), ("adamw", pdt.optim.AdamW)):
        opt = cli.make_optimizer(cli.build_parser().parse_args(["--optimizer", name, "--amsgrad"]), p)
        assert type(opt) is cls and opt.param_groups[0]["amsgrad"] is True
    assert cli.make_optimizer(cli.build_parser().parse_args(["--optimizer", "adamw"]), p).param_groups[0]["amsgrad"] is False
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train_mnist.py"), "--optimizer", "sgd", "--amsgrad"],
                         capture_output=True, text=True, timeout=60, cwd=ROOT)
    assert out.returncode != 0 and "--amsgrad applies to Adam and AdamW only" in out.stderr, out.stderr[-2000:]


@pytest.mark.parametrize("cls", [pdt.optim.Adam, pdt.optim.AdamW])
def test_sync_lr_refuses_a_replay_after_amsgrad_changed(cls):
    """A captured step baked the kernel (with or without the maximum) into the graph: flipping amsgrad afterwards is refused."""
    opt = cls([torch.zeros(3, requires_grad=True)], lr=0.1)
    opt._record_captured_hyper()
    opt.sync_lr()
    opt.param_groups[0]["lr"] = 0.05
    opt.sync_lr()   # lr may change
    opt.param_groups[0]["amsgrad"] = True
    with pytest.raises(RuntimeError, match="'amsgrad' of param_groups\\[0\\] changed from False to True"):
        opt.sync_lr()


def test_train_script_adamw_amsgrad_checkpoint_and_resume(tmp_path):
    ck = str(tmp_path / "amsgrad.pt")
    base = [sys.executable, os.path.join(ROOT, "train_mnist.py"), "-g", "2", "--backend", "gloo", "--optimizer", "adamw", "--amsgrad",
            "--lr", "1e-3", "--steps", "3", "--samples", "600", "--log-interval", "3"]
    a = subprocess.run(base + ["--epochs", "1", "--checkpoint", ck], capture_output=True, text=True, timeout=240, cwd=ROOT)
    assert a.returncode == 0 and os.path.exists(ck), a.stderr[-2000:]
    saved = torch.load(ck, map_location="cpu", weights_only=False)["optimizer"]
    assert saved["param_groups"][0]["amsgrad"] is True and saved["param_groups"][0]["decoupled_weight_decay"] is True
    assert all(float(st["step"]) == 3.0 and "max_exp_avg_sq" in st for st in saved["state"].values())
    assert all(bool((st["max_exp_avg_sq"] >= st["exp_avg_sq"]).all()) for st in saved["state"].values())
    b = subprocess.run(base + ["--epochs", "2", "--resume", ck], capture_output=True, text=True, timeout=240, cwd=ROOT)
    assert b.returncode == 0, b.stderr[-2000:]
    assert "Resumed from" in b.stdout and "Epoch [2/2], Step [3/3]" in b.stdout and "Epoch [1/2]" not in b.stdout


# =====================================================================================================================
# GPU
# =====================================================================================================================
def _dev():
    return torch.device("cuda", 0)


def _amsgrad_f64(p, grads, lr, beta1, beta2, eps, wd, decoupled, maximize):
    """AMSGrad in float64 (the oracle of the kernel's arithmetic): p, exp_avg, exp_avg_sq, max_exp_avg_sq after the steps."""
    m, v, vmax = torch.zeros_like(p), torch.zeros_like(p), torch.zeros_like(p)
    for step, g in enumerate(grads, 1):
        g = -g if maximize else g
        if wd:
            if decoupled:
                p = p * (1 - lr * wd)
            else:
                g = g + wd * p
        m = m + (1 - beta1) * (g - m)
        v = beta2 * v + (1 - beta2) * g * g
        vmax = torch.maximum(vmax, v)
        p = p - (lr / (1 - beta1 ** step)) * m / (vmax.sqrt() / (1 - beta2 ** step) ** 0.5 + eps)
    return p, m, v, vmax


@pytest.mark.gpu
@pytest.mark.parametrize("ours,theirs", PAIRS)
@pytest.mark.parametrize("kw", [dict(weight_decay=0.0), dict(weight_decay=1e-2), dict(weight_decay=1e-2, maximize=True)])
@pytest.mark.parametrize("tables", [1, 2])
def test_kernel_matches_torch_and_float64_over_ten_steps(ours, theirs, kw, tables):
    """Ten AMSGrad steps of the multi-tensor kernel against torch's single-tensor AMSGrad and a float64 oracle.  The gradients
    shrink from step to step, so exp_avg_sq falls below its running maximum in most elements and the denominator comes from the
    maximum.  tables=2: 50 tensors, more than one table of 48 holds."""
    from pytorch_distributed_train_b200 import _C

    torch.manual_seed(7)
    shapes = CONVNET_SIZES + [(100003,)]
    if tables == 2:
        shapes = (CONVNET_SIZES * 5)[:49] + [(100003,)]
    pa = [torch.randn(s, device=_dev()).requires_grad_() for s in shapes]
    pb = [p.detach().clone().requires_grad_() for p in pa]
    init = [p.detach().double() for p in pa]
    a = ours(pa, lr=1e-2, amsgrad=True, **kw)
    b = theirs(pb, lr=1e-2, amsgrad=True, foreach=False, **kw)
    # from 10 down to 10^-3.5: also with Adam's coupled weight decay (g + wd·p) the late gradients stay below sqrt(exp_avg_sq)
    grads = [[torch.randn(s, device=_dev()) * 10 ** (1 - i / 2) for s in shapes] for i in range(10)]
    launches = 0
    for gs in grads:
        for p, q, g in zip(pa, pb, gs):
            p.grad, q.grad = g.clone(), g.clone()
        c0 = _C.kernel_launch_count()
        a.step()
        launches += _C.kernel_launch_count() - c0
        b.step()
    assert launches == 10 * tables, f"one multi-tensor launch per table of up to 48 tensors per step ({launches})"
    wd, decoupled = kw["weight_decay"], ours is pdt.optim.AdamW
    above = total = 0
    for i, (p, q) in enumerate(zip(pa, pb)):
        sa, sb = a.state[p], b.state[q]
        assert set(sa) == set(sb) == {"step", "exp_avg", "exp_avg_sq", "max_exp_avg_sq"}
        assert sa["step"].is_cuda and sa["step"].dtype == torch.float32 and sa["step"].item() == 10.0 == sb["step"].item()
        for name in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"):
            assert torch.allclose(sa[name], sb[name], rtol=1e-5, atol=1e-7), (i, name, (sa[name] - sb[name]).abs().max().item())
        assert torch.allclose(p, q, rtol=1e-5, atol=1e-7), (i, (p - q).abs().max().item())
        above += int((sa["max_exp_avg_sq"] > sa["exp_avg_sq"]).sum())
        total += p.numel()
        ref = _amsgrad_f64(init[i], [gs[i].double() for gs in grads], 1e-2, 0.9, 0.999, 1e-8, wd, decoupled, kw.get("maximize", False))
        # relative to the largest magnitude the value was formed from (test_adam.py's oracle comparison)
        g_max = torch.stack([gs[i].abs() for gs in grads]).amax(0).double()
        for name, x, y, scale in (("p", p, ref[0], init[i].abs()), ("exp_avg", sa["exp_avg"], ref[1], g_max),
                                  ("exp_avg_sq", sa["exp_avg_sq"], ref[2], ref[2].abs()),
                                  ("max_exp_avg_sq", sa["max_exp_avg_sq"], ref[3], ref[3].abs())):
            err = (x.double() - y).abs()
            assert bool((err <= 1e-5 * torch.maximum(y.abs(), scale) + 1e-7).all()), (i, name, err.max().item())
    assert above > 0.8 * total, f"the maximum must be exercised: max_exp_avg_sq > exp_avg_sq in {above} of {total} elements"


@pytest.mark.gpu
def test_nan_gradient_stays_in_its_element_as_in_torch():
    """torch.maximum keeps a NaN (fmaxf would drop it): a NaN gradient leaves NaN in that element's max_exp_avg_sq and parameter for
    good, and every other element is what a run without the NaN gives."""
    torch.manual_seed(8)
    shapes = [(300,), (17, 5)]
    runs = []
    for poison in (True, False):
        ours = [torch.randn(s, device=_dev(), generator=torch.Generator(device=_dev()).manual_seed(1)).requires_grad_() for s in shapes]
        theirs = [p.detach().clone().requires_grad_() for p in ours]
        a = pdt.optim.AdamW(ours, lr=1e-2, amsgrad=True)
        b = torch.optim.AdamW(theirs, lr=1e-2, amsgrad=True, foreach=False)
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
    assert torch.isnan(a.state[ours[0]]["max_exp_avg_sq"][123]) and torch.isnan(ours[0][123])
    for p, q, c in zip(ours, theirs, clean):
        for x, y in [(p, q)] + [(a.state[p][k], b.state[q][k]) for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")]:
            assert torch.equal(torch.isnan(x), torch.isnan(y))
            assert torch.allclose(x, y, rtol=1e-5, atol=1e-7, equal_nan=True)
        keep = ~torch.isnan(p)
        assert int((~keep).sum()) == (1 if p is ours[0] else 0)
        assert torch.equal(p[keep], c[keep]), "the other elements must be unaffected"
        assert torch.equal(a.state[p]["max_exp_avg_sq"][keep], ca.state[c]["max_exp_avg_sq"][keep])


@pytest.mark.gpu
def test_captured_amsgrad_step_replays_with_a_schedule():
    """One AMSGrad adam_step in a CUDA graph, replayed 20 times with shrinking gradients and the learning rate changed through
    sync_lr after 10: the same as 20 eager torch steps, and the step count reads 20."""
    from pytorch_distributed_train_b200 import ops

    torch.manual_seed(6)
    shapes = [(300,), (17, 5), (1,)]
    pa = [torch.randn(s, device=_dev()).requires_grad_() for s in shapes]
    pb = [p.detach().clone().requires_grad_() for p in pa]
    base = [torch.randn_like(p) for p in pa]
    for p, q, g in zip(pa, pb, base):
        p.grad, q.grad = g.clone(), g.clone()
    a = pdt.optim.AdamW(pa, lr=1e-2, amsgrad=True, capturable=True)
    b = torch.optim.AdamW(pb, lr=1e-2, amsgrad=True, foreach=False)
    # everything a captured step reads must exist before the capture: the state, the learning-rate scalar, the kernel's scratch
    for p in pa:
        a._state(p, True)
    a._lr_tensor(0, a.param_groups[0], _dev())
    z = torch.zeros(4, device=_dev())
    ops.adam_step([z.clone()], [z.clone()], [z.clone()], [z.clone()], [torch.zeros((), device=_dev())], lr=0.0, max_exp_avg_sqs=[z.clone()])
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
        for p, q, g in zip(pa, pb, base):
            p.grad.copy_(g * 0.5 ** r)   # in place: the graph reads these tensors
            q.grad.copy_(g * 0.5 ** r)
        graph.replay()
        b.step()
    torch.cuda.synchronize()
    for p, q in zip(pa, pb):
        sa, sb = a.state[p], b.state[q]
        assert sa["step"].item() == 20.0
        assert torch.allclose(p, q, rtol=1e-5, atol=1e-7), (p - q).abs().max().item()
        for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"):
            assert torch.allclose(sa[k], sb[k], rtol=1e-5, atol=1e-7), k
        assert bool((sa["max_exp_avg_sq"] > sa["exp_avg_sq"]).all())


def _convnet_batch(s, n=100):
    g = torch.Generator(device=_dev()).manual_seed(s)
    return torch.rand(n, 1, 28, 28, device=_dev(), generator=g), torch.randint(0, 10, (n,), device=_dev(), generator=g)


@pytest.mark.gpu
@pytest.mark.parametrize("cls,clip", [(pdt.optim.Adam, False), (pdt.optim.AdamW, False), (pdt.optim.AdamW, True)])
def test_amsgrad_rider_rides_on_the_last_backward_kernel(cls, clip):
    """AdamW(amsgrad=True).ride_on_backward: the layer-1 backward kernel applies the AMSGrad update of all ten parameters
    (AmsgradRider, or ClipRider<AmsgradRider> with clip=); parameters and the four state tensors follow the separate kernel (after
    clip_grad_norm_ with clip=).  beta2 = 0.6 lets exp_avg_sq fall below its maximum within four steps."""
    from pytorch_distributed_train_b200 import _C
    from pytorch_distributed_train_b200.nn.utils import clip_grad_norm_
    from pytorch_distributed_train_b200.ops import functional as OF

    torch.manual_seed(4)
    a = pdt.models.ConvNet(fused=True).to(_dev())
    b = pdt.models.ConvNet(fused=True).to(_dev())
    b.load_state_dict(a.state_dict())
    oa = cls(a.parameters(), 1e-3, betas=(0.9, 0.6), weight_decay=1e-2, amsgrad=True)
    ob = cls(b.parameters(), 1e-3, betas=(0.9, 0.6), weight_decay=1e-2, amsgrad=True)
    crit = pdt.nn.CrossEntropyLoss()
    max_norm = 0.05
    norm_out = torch.zeros((), device=_dev())
    # the clipping paths fold the norm in different orders: the coefficients may differ in the last bit (test_clip_grad.py)
    skip = NOISE if clip else ()
    assert oa.ride_on_backward(a, clip=(max_norm, 2.0, norm_out) if clip else None) and OF._sgd_rider.owner is oa
    try:
        for s in range(4):
            x, t = _convnet_batch(s)
            before = _C.kernel_launch_count()
            oa.zero_grad()
            la = crit(a(x), t)
            with OF.sgd_rider_enabled():
                la.backward()
            assert oa._rode, "the backward kernel should have applied the update"
            oa.step()
            riding = _C.kernel_launch_count() - before
            before = _C.kernel_launch_count()
            ob.zero_grad()
            crit(b(x), t).backward()
            if clip:
                nb = clip_grad_norm_(b.parameters(), max_norm)
            ob.step()
            separate = _C.kernel_launch_count() - before
            assert riding < separate, (riding, separate)
            if clip:
                torch.cuda.synchronize()
                assert nb.item() > max_norm, "clipping must engage"
                assert abs(norm_out.item() - nb.item()) <= 1e-4 * nb.item(), (norm_out.item(), nb.item())
            for (n1, p1), p2 in zip(a.named_parameters(), b.parameters()):
                if n1 not in skip:
                    assert torch.allclose(p1, p2, atol=1e-6, rtol=1e-5), (s, n1, (p1 - p2).abs().max().item())
        above = total = 0
        for (n1, p1), p2 in zip(a.named_parameters(), b.parameters()):
            s1, s2 = oa.state[p1], ob.state[p2]
            assert set(s1) == set(s2) == {"step", "exp_avg", "exp_avg_sq", "max_exp_avg_sq"}
            assert s1["step"].item() == s2["step"].item() == 4.0
            above += int((s1["max_exp_avg_sq"] > s1["exp_avg_sq"]).sum())
            total += p1.numel()
            if n1 in skip:
                continue
            assert torch.allclose(s1["exp_avg"], s2["exp_avg"], atol=1e-7, rtol=1e-5), n1
            for k in ("exp_avg_sq", "max_exp_avg_sq"):
                assert torch.allclose(s1[k], s2[k], atol=1e-9, rtol=1e-5), (n1, k)
        assert above > 0.05 * total, f"the maximum must be exercised ({above} of {total} elements)"
    finally:
        oa.stop_riding()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain", "clip", "accumulate"])
def test_graphed_step_with_amsgrad_is_three_launches_per_batch_and_follows_torch(mode):
    """engine.GraphedTrainStep with pdt.optim.AdamW(amsgrad=True) on one GPU: the update rides on the last backward kernel, so a
    replay is 3 launches (also with max_grad_norm, 3k with accumulation_steps=k), and 20 replays follow an eager loop with
    torch.optim.AdamW(amsgrad=True) within bench.py's verification tolerance."""
    from mp_helpers import free_port

    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    k = 2 if mode == "accumulate" else 1
    max_norm = 1.0 if mode == "clip" else None
    torch.cuda.set_device(0)
    pdt.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{free_port()}", world_size=1, rank=0)
    try:
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(_dev())
        opt = pdt.optim.AdamW(model.parameters(), 1e-3, amsgrad=True)
        ddp = pdt.DistributedDataParallel(model, device_ids=[0])
        crit = pdt.nn.CrossEntropyLoss()
        batches = [_convnet_batch(90 + i, 100 * k) for i in range(4)]
        step = GraphedTrainStep(ddp, crit, opt, batches[0], warmup=3, max_grad_norm=max_norm, accumulation_steps=k)
        assert step.kernels_per_replay == 3 * k, step.kernels_per_replay
        # the reference starts where the engine's eager warm-up steps left the model and the optimizer
        ref = pdt.models.ConvNet().to(_dev())
        ref.load_state_dict(model.state_dict())
        ropt = torch.optim.AdamW(ref.parameters(), 1e-3, amsgrad=True, foreach=False)
        ropt.load_state_dict(copy.deepcopy(opt.state_dict()))   # torch would otherwise share our state tensors
        assert ropt.param_groups[0]["amsgrad"] is True
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
        assert all("max_exp_avg_sq" in st for st in opt.state.values())
        # bench.py's verification metric (max |ours − reference| / max |reference| over the flat vector, tolerance 2e-2)
        keep = [(p, q) for (n, p), q in zip(model.named_parameters(), ref.parameters()) if n not in NOISE]
        ours_flat = torch.cat([p.detach().reshape(-1) for p, _ in keep])
        ref_flat = torch.cat([q.detach().reshape(-1) for _, q in keep])
        err = (ours_flat - ref_flat).abs().max().item() / ref_flat.abs().max().item()
        assert err < 2e-2, err
    finally:
        pdt.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("direction", ["torch_to_pdt", "pdt_to_torch"])
def test_state_dict_with_max_exp_avg_sq_moves_between_torch_and_pdt_on_cuda(direction):
    torch.manual_seed(3)
    shapes = [(5, 3), (7,), (4, 4)]
    pa = [torch.randn(s, device=_dev()).requires_grad_() for s in shapes]
    pb = [p.detach().clone().requires_grad_() for p in pa]
    def theirs(params, **kw):
        return torch.optim.Adam(params, foreach=False, **kw)

    src_cls, dst_cls = (theirs, pdt.optim.Adam) if direction == "torch_to_pdt" else (pdt.optim.Adam, theirs)
    src = src_cls(pa, lr=1e-2, weight_decay=1e-2, amsgrad=True)
    g = torch.Generator(device=_dev()).manual_seed(4)
    for s in range(3):
        for p in pa:
            p.grad = torch.randn(p.shape, device=_dev(), generator=g) * 0.3 ** s
        src.step()
    with torch.no_grad():
        for p, q in zip(pa, pb):
            q.copy_(p)
    dst = dst_cls(pb, lr=5.0)
    dst.load_state_dict(copy.deepcopy(src.state_dict()))
    assert dst.param_groups[0]["amsgrad"] is True and dst.param_groups[0]["lr"] == 1e-2
    for p, q in zip(pa, pb):
        assert torch.equal(dst.state[q]["max_exp_avg_sq"].to(_dev()), src.state[p]["max_exp_avg_sq"])
        assert float(dst.state[q]["step"]) == 3.0
    for s in range(3):
        for p, q in zip(pa, pb):
            p.grad = torch.randn(p.shape, device=_dev(), generator=g) * 0.1
            q.grad = p.grad.clone()
        src.step()
        dst.step()
    for p, q in zip(pa, pb):
        assert float(src.state[p]["step"]) == float(dst.state[q]["step"]) == 6.0
        assert torch.allclose(p, q, rtol=1e-5, atol=1e-7), (p - q).abs().max().item()
        for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"):
            assert torch.allclose(src.state[p][k], dst.state[q][k], rtol=1e-5, atol=1e-7), k


@pytest.mark.gpu
def test_fused_true_with_amsgrad_runs_the_kernel():
    """Adam(fused=True, amsgrad=True) takes the multi-tensor kernel (one launch per step), as torch's fused Adam accepts it."""
    from pytorch_distributed_train_b200 import _C

    torch.manual_seed(9)
    pa = [torch.randn(s, device=_dev()).requires_grad_() for s in [(64, 3), (1000,)]]
    pb = [p.detach().clone().requires_grad_() for p in pa]
    a = pdt.optim.Adam(pa, lr=1e-2, amsgrad=True, fused=True)
    b = torch.optim.Adam(pb, lr=1e-2, amsgrad=True, fused=True)
    for s in range(3):
        for p, q in zip(pa, pb):
            p.grad = torch.randn_like(p) * 0.2 ** s
            q.grad = p.grad.clone()
        c0 = _C.kernel_launch_count()
        a.step()
        assert _C.kernel_launch_count() - c0 == 1
        b.step()
    # torch's fused kernel forms 1 − β2 in fp32 (1 − fp32(0.999) is 1.3e-5 below fp32(0.001)); ours follows the single-tensor
    # arithmetic, in which it comes from double
    for p, q in zip(pa, pb):
        assert torch.allclose(p, q, rtol=1e-5, atol=1e-6), (p - q).abs().max().item()
        assert torch.allclose(a.state[p]["max_exp_avg_sq"], b.state[q]["max_exp_avg_sq"], rtol=5e-5, atol=1e-9)
