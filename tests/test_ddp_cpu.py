"""DDP end-to-end on the CPU backend, world_size=2 (BASELINE.json config 1), with
torch DDP + gloo as the oracle."""
import io
import os

import pytest
import torch
import torch.nn as nn

import pytorch_distributed_train_b200 as pdt
from mp_helpers import free_port, run_ranks

dist = pdt.distributed


def _data(rank, step, bs=8):
    g = torch.Generator().manual_seed(1000 * step + rank)
    return torch.rand(bs, 1, 28, 28, generator=g), torch.randint(0, 10, (bs,), generator=g)


def _train_ours(rank, world, steps, syncbn=False, **ddp_kw):
    torch.manual_seed(0)
    model = pdt.models.ConvNet()
    if syncbn:
        model = pdt.SyncBatchNorm.convert_sync_batchnorm(model)
    opt = pdt.optim.SGD(model.parameters(), 0.05)  # optimizer built before wrapping, like the reference
    ddp = pdt.DistributedDataParallel(model, **ddp_kw)
    crit = pdt.nn.CrossEntropyLoss()
    losses = []
    for s in range(steps):
        x, y = _data(rank, s)
        loss = crit(ddp(x), y)
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    return ddp, losses


def _train_torch(rank, world, steps, port):
    import torch.distributed as td

    td.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", world_size=world, rank=rank)
    torch.manual_seed(0)
    model = pdt.models.ConvNet(fused=False)
    opt = torch.optim.SGD(model.parameters(), 0.05)
    ddp = nn.parallel.DistributedDataParallel(model)
    crit = nn.CrossEntropyLoss()
    losses = []
    for s in range(steps):
        x, y = _data(rank, s)
        loss = crit(ddp(x), y)
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    sd = {k: v.clone() for k, v in ddp.state_dict().items()}
    grads = [p.grad.clone() for p in ddp.parameters()]
    td.destroy_process_group()
    return losses, sd, grads


def _vs_torch(rank, world, port):
    steps = 4
    ddp, losses = _train_ours(rank, world, steps)
    ref_losses, ref_sd, ref_grads = _train_torch(rank, world, steps, port)
    sd = ddp.state_dict()
    assert list(sd.keys()) == list(ref_sd.keys()), "state_dict keys must carry the module. prefix like torch DDP"
    assert all(k.startswith("module.") for k in sd)
    for k in sd:
        assert torch.allclose(sd[k].float(), ref_sd[k].float(), atol=1e-5, rtol=1e-4), k
    for p, g in zip(ddp.parameters(), ref_grads):
        assert torch.allclose(p.grad, g, atol=1e-6, rtol=1e-4)
    assert torch.allclose(torch.tensor(losses), torch.tensor(ref_losses), atol=1e-5)
    info = ddp._get_ddp_logging_data()
    flat = torch.cat([p.detach().reshape(-1) for p in ddp.parameters()])
    pre = ddp.module.layer1[1].running_mean.clone()
    ddp._sync_buffers()  # what the next training forward does first
    return {"losses": losses, "param_sum": flat.double().sum().item(), "info": info,
            "bn_mean_before_sync": pre, "bn_mean": ddp.module.layer1[1].running_mean.clone()}


def test_matches_torch_ddp_gloo():
    res = run_ranks(_vs_torch, 2, free_port())
    a, b = res
    assert a["param_sum"] == b["param_sum"], "parameters must be identical across ranks after every step"
    assert not torch.equal(a["bn_mean_before_sync"], b["bn_mean_before_sync"])  # local batches differ
    assert torch.equal(a["bn_mean"], b["bn_mean"]), "BN buffers follow rank 0 (C4 semantics)"
    assert torch.equal(a["bn_mean"], a["bn_mean_before_sync"])
    info = a["info"]
    assert info["bucket_sizes"] == [116136] and info["total_parameter_size_bytes"] == 116136
    assert info["has_rebuilt_buckets"] and info["num_parameter_tensors"] == 10
    # grad-ready order observed for the reference model
    assert info["grad_ready_order"] == [9, 8, 6, 7, 4, 5, 2, 3, 0, 1]
    assert info["bucket_indices"] == [[9, 8, 6, 7, 4, 5, 2, 3, 0, 1]]
    assert info["world_size"] == 2 and info["module_name"] == "ConvNet"


def _grad_is_mean(rank, world):
    torch.manual_seed(0)
    model = pdt.models.ConvNet()
    ddp = pdt.DistributedDataParallel(model, bucket_cap_mb=0.03, first_bucket_cap_mb=0.001)
    crit = nn.CrossEntropyLoss()
    x, y = _data(rank, 0)
    crit(ddp(x), y).backward()
    got = [p.grad.clone() for p in ddp.parameters()]
    assert ddp.reducer.grads_are_views()
    # local gradients of every rank, computed without DDP on an identical copy
    locals_ = []
    for r in range(world):
        torch.manual_seed(0)
        m = pdt.models.ConvNet()
        m.load_state_dict(ddp.module.state_dict())
        # undo this step's running-stat update so each replica sees the same pre-step buffers
        xr, yr = _data(r, 0)
        m.train()
        crit(m(xr), yr).backward()
        locals_.append([p.grad.clone() for p in m.parameters()])
    for i, g in enumerate(got):
        mean = sum(l[i] for l in locals_) / world
        assert torch.allclose(g, mean, atol=1e-6, rtol=1e-4), i
    return ddp._get_ddp_logging_data()["bucket_sizes"]


def test_gradients_are_mean_of_local_gradients_multi_bucket():
    res = run_ranks(_grad_is_mean, 2)
    assert res[0] == res[1] and len(res[0]) > 1, f"expected several buckets, got {res[0]}"
    assert sum(res[0]) == 116136


def _no_sync(rank, world):
    torch.manual_seed(0)
    ddp = pdt.DistributedDataParallel(pdt.models.ConvNet())
    crit = nn.CrossEntropyLoss()
    x0, y0 = _data(rank, 0)
    x1, y1 = _data(rank, 1)
    with ddp.no_sync():
        crit(ddp(x0), y0).backward()
    local_only = ddp.module.fc.bias.grad.clone()
    crit(ddp(x1), y1).backward()
    synced = ddp.module.fc.bias.grad.clone()
    gathered = dist.all_gather_object((local_only, synced))
    return gathered


def test_no_sync_accumulates_then_reduces():
    res = run_ranks(_no_sync, 2)
    (l0, s0), (l1, s1) = res[0]
    assert not torch.allclose(l0, l1), "inside no_sync gradients stay local"
    assert torch.allclose(s0, s1, atol=1e-7), "first synced backward reduces the accumulated gradients"


def _hook(rank, world):
    from pytorch_distributed_train_b200.parallel import comm_hooks

    torch.manual_seed(0)
    ddp = pdt.DistributedDataParallel(pdt.models.ConvNet())
    seen = []

    def hook(state, bucket):
        seen.append((bucket.index(), bucket.is_last(), bucket.buffer().numel(), len(bucket.gradients()), len(bucket.parameters())))
        return comm_hooks.allreduce_hook(state, bucket)

    ddp.register_comm_hook(None, hook)
    crit = nn.CrossEntropyLoss()
    x, y = _data(rank, 0)
    crit(ddp(x), y).backward()
    g = ddp.module.fc.weight.grad.clone()
    try:
        ddp.register_comm_hook(None, hook)
        twice = False
    except RuntimeError:
        twice = True
    return seen, g, twice


def test_comm_hook_sees_one_bucket_and_averages():
    res = run_ranks(_hook, 2)
    seen, g0, twice = res[0]
    assert twice
    assert len(seen) == 1 and seen[0][0] == 0 and seen[0][1] is True and seen[0][3] == 10
    assert seen[0][2] >= 29034
    assert torch.allclose(g0, res[1][1], atol=1e-7)


def _compress_hooks(rank, world):
    from pytorch_distributed_train_b200.parallel import comm_hooks

    out = []
    for hook in (comm_hooks.bf16_compress_hook, comm_hooks.fp16_compress_hook):
        torch.manual_seed(0)
        ddp = pdt.DistributedDataParallel(pdt.models.ConvNet())
        ddp.register_comm_hook(None, hook)
        x, y = _data(rank, 0)
        nn.CrossEntropyLoss()(ddp(x), y).backward()
        out.append(ddp.module.fc.weight.grad.clone())
    torch.manual_seed(0)
    ddp = pdt.DistributedDataParallel(pdt.models.ConvNet())
    x, y = _data(rank, 0)
    nn.CrossEntropyLoss()(ddp(x), y).backward()
    out.append(ddp.module.fc.weight.grad.clone())
    return out


def test_compression_hooks_close_to_exact():
    res = run_ranks(_compress_hooks, 2)
    bf, fp, exact = res[0]
    assert torch.allclose(fp, exact, atol=2e-3, rtol=2e-2)
    assert torch.allclose(bf, exact, atol=1e-2, rtol=5e-2)


class _Branchy(nn.Module):
    def __init__(self):
        super().__init__()
        self.a = nn.Linear(4, 4)
        self.b = nn.Linear(4, 4)
        self.never = nn.Linear(4, 4)

    def forward(self, x, use_b):
        return self.b(x) if use_b else self.a(x)


def _unused(rank, world):
    torch.manual_seed(0)
    ddp = pdt.DistributedDataParallel(_Branchy(), find_unused_parameters=True)
    x = torch.ones(2, 4) * (rank + 1)
    ddp(x, use_b=(rank == 1)).sum().backward()
    m = ddp.module
    return (m.a.weight.grad.clone(), m.b.weight.grad.clone(), m.never.weight.grad is None)


def test_find_unused_parameters():
    res = run_ranks(_unused, 2)
    (a0, b0, n0), (a1, b1, n1) = res
    assert n0 and n1, "a parameter unused on every rank keeps grad=None"
    assert torch.allclose(a0, a1) and torch.allclose(b0, b1)
    assert torch.allclose(a0, torch.ones(4, 4) * 2 * 1 / 2), "rank0 used a with x=1, rank1 contributed zeros"
    assert torch.allclose(b0, torch.ones(4, 4) * 2 * 2 / 2)


def _mismatch(rank, world):
    torch.manual_seed(0)
    model = nn.Linear(4, 4 if rank == 0 else 5)
    try:
        pdt.DistributedDataParallel(model)
    except RuntimeError as e:
        return str(e)
    return ""


def test_mismatched_models_raise_on_every_rank():
    res = run_ranks(_mismatch, 2)
    assert all("params not equal across ranks" in r or "same model" in r for r in res), res


def _init_broadcast(rank, world):
    torch.manual_seed(rank)  # deliberately different init per rank
    ddp = pdt.DistributedDataParallel(pdt.models.ConvNet())
    return torch.cat([p.detach().reshape(-1) for p in ddp.parameters()]).sum().item()


def test_init_broadcast_from_rank0():
    a, b = run_ranks(_init_broadcast, 2)
    assert a == b


def _syncbn(rank, world):
    torch.manual_seed(0)
    bn = pdt.SyncBatchNorm(6)
    g = torch.Generator().manual_seed(7)
    full = torch.randn(10, 6, 5, 5, generator=g)
    # uneven split: rank 0 gets 7 samples, rank 1 gets 3 (count-weighting must hold)
    mine = full[:7] if rank == 0 else full[7:]
    x = mine.clone().requires_grad_(True)
    out = bn(x)
    wgt = torch.arange(out.numel(), dtype=torch.float32).view_as(out) / out.numel()
    # loss over the *global* batch = sum of per-rank pieces
    (out * wgt).sum().backward()
    ref_bn = nn.BatchNorm2d(6)
    xf = full.clone().requires_grad_(True)
    ref_out = ref_bn(xf)
    sl = slice(0, 7) if rank == 0 else slice(7, 10)
    w_full = torch.zeros_like(ref_out)
    w_full[sl] = wgt
    # every rank's backward in the sync version only sees its own loss piece, but dx depends on
    # the global Σdy; emulate by summing both ranks' weights
    other = torch.arange((10 - mine.shape[0]) * 6 * 25, dtype=torch.float32).view(-1, 6, 5, 5) / ((10 - mine.shape[0]) * 6 * 25)
    w_full[slice(7, 10) if rank == 0 else slice(0, 7)] = other
    (ref_out * w_full).sum().backward()
    assert torch.allclose(out, ref_out[sl], atol=1e-5), "forward must use global statistics"
    assert torch.allclose(x.grad, xf.grad[sl], atol=1e-5), "dx must use global Σdy, Σdy·x̂"
    assert torch.allclose(bn.running_mean, ref_bn.running_mean, atol=1e-6)
    assert torch.allclose(bn.running_var, ref_bn.running_var, atol=1e-5)
    assert int(bn.num_batches_tracked) == 1
    # dγ/dβ are local sums; DDP (or a manual allreduce) completes them
    gw = bn.weight.grad.clone()
    dist.all_reduce(gw)
    assert torch.allclose(gw, ref_bn.weight.grad, atol=1e-4)
    bn.eval()
    assert torch.allclose(bn(mine), ref_bn.eval()(mine), atol=1e-5)
    return True


def test_syncbn_matches_global_batchnorm_uneven_batches():
    assert all(run_ranks(_syncbn, 2))


def test_convert_sync_batchnorm_shares_tensors():
    m = pdt.models.ConvNet()
    w, rm, nbt = m.layer1[1].weight, m.layer1[1].running_mean, m.layer1[1].num_batches_tracked
    c = pdt.SyncBatchNorm.convert_sync_batchnorm(m)
    assert isinstance(c.layer1[1], pdt.SyncBatchNorm) and isinstance(c.layer2[1], pdt.SyncBatchNorm)
    assert c.layer1[1].weight is w and c.layer1[1].running_mean is rm and c.layer1[1].num_batches_tracked is nbt
    assert list(c.state_dict().keys()) == list(pdt.models.ConvNet().state_dict().keys())
    # world of one / uninitialised: behaves like plain BN
    x = torch.randn(4, 1, 28, 28)
    torch.manual_seed(0)
    a = c(x)
    assert a.shape == (4, 10)


def _syncbn_ddp(rank, world):
    ddp, losses = _train_ours(rank, world, 3, syncbn=True)
    sd = ddp.state_dict()
    return losses, sd["module.layer2.1.running_var"].clone(), torch.cat([p.detach().reshape(-1) for p in ddp.parameters()]).sum().item()


def test_syncbn_under_ddp_keeps_ranks_identical():
    (l0, v0, p0), (l1, v1, p1) = run_ranks(_syncbn_ddp, 2)
    assert torch.equal(v0, v1) and p0 == p1
    assert all(torch.isfinite(torch.tensor(l0 + l1)))


def _join(rank, world):
    torch.manual_seed(0)
    ddp = pdt.DistributedDataParallel(pdt.models.ConvNet())
    opt = pdt.optim.SGD(ddp.parameters(), 0.05)
    crit = nn.CrossEntropyLoss()
    n_steps = 2 if rank == 0 else 4
    with ddp.join():
        for s in range(n_steps):
            x, y = _data(rank, s)
            loss = crit(ddp(x), y)
            opt.zero_grad()
            loss.backward()
            opt.step()
    return torch.cat([p.detach().reshape(-1) for p in ddp.parameters()]).sum().item()


def test_join_uneven_inputs():
    a, b = run_ranks(_join, 2)
    assert a == b


def test_state_dict_roundtrip_and_pickle_keys():
    pdt.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{free_port()}", world_size=1, rank=0)
    try:
        ddp = pdt.DistributedDataParallel(pdt.models.ConvNet())
        sd = ddp.state_dict()
        assert "module.fc.weight" in sd and "module.layer1.1.num_batches_tracked" in sd
        buf = io.BytesIO()
        torch.save(sd, buf)
        buf.seek(0)
        ddp2 = pdt.DistributedDataParallel(pdt.models.ConvNet())
        ddp2.load_state_dict(torch.load(buf))
        assert torch.equal(ddp2.module.fc.weight, ddp.module.fc.weight)
        with pytest.raises(RuntimeError):
            pdt.DistributedDataParallel(nn.ReLU())
    finally:
        pdt.destroy_process_group()


def test_requires_process_group():
    with pytest.raises(RuntimeError):
        pdt.DistributedDataParallel(pdt.models.ConvNet())


def _fused_opt(rank, world, momentum):
    """optim.SGD.fuse_with_ddp: the optimizer owns the gradient allreduce; results must equal the
    reducer-driven path step for step (protocol test on the CPU backend; the one-kernel version is
    tests/test_gpu_multigpu.py::test_fused_allreduce_sgd)."""
    out = []
    for fuse in (False, True):
        torch.manual_seed(0)
        model = pdt.models.ConvNet()
        opt = pdt.optim.SGD(model.parameters(), 0.05, momentum=momentum, weight_decay=1e-3 if momentum else 0.0)
        ddp = pdt.DistributedDataParallel(model)
        if fuse:
            opt.fuse_with_ddp(ddp)
        crit = pdt.nn.CrossEntropyLoss()
        for s in range(6):
            x, y = _data(rank, s)
            loss = crit(ddp(x), y)
            opt.zero_grad()
            loss.backward()
            opt.step()
        assert bool(opt._fused_active) == fuse
        if fuse:
            assert ddp.reducer.fused_sgd and ddp._get_ddp_logging_data()["params_flattened"]
            assert ddp._get_ddp_logging_data()["reduce_chunks"] == 2  # fc | bn2+conv2+bn1+conv1 (32 KiB granularity; the 1.8 KB tail rides with the chunk before it)
            # gradients still read as the averaged gradient after step()
            g = [p.grad.clone() for p in ddp.parameters()]
            assert all(torch.isfinite(t).all() for t in g)
        out.append(torch.cat([p.detach().flatten() for p in ddp.parameters()]))
    return out


@pytest.mark.parametrize("momentum", [0.0, 0.9])
def test_optimizer_fused_allreduce_matches_reducer_path(momentum):
    for plain, fused in run_ranks(_fused_opt, 2, momentum):
        assert torch.allclose(plain, fused, rtol=1e-5, atol=1e-6)


def _ckpt(rank, world, path, fuse):
    """Train 2 steps, checkpoint, train 2 more — versus a fresh process state restored from the checkpoint and
    trained for the same 2 steps: identical parameters and momentum."""
    def fresh():
        torch.manual_seed(0)
        model = pdt.models.ConvNet()
        opt = pdt.optim.SGD(model.parameters(), 0.05, momentum=0.9)
        ddp = pdt.DistributedDataParallel(model)
        if fuse:
            opt.fuse_with_ddp(ddp)
        return ddp, opt

    def train(ddp, opt, steps):
        crit = pdt.nn.CrossEntropyLoss()
        for s in steps:
            x, y = _data(rank, s)
            loss = crit(ddp(x), y)
            opt.zero_grad()
            loss.backward()
            opt.step()

    ddp, opt = fresh()
    train(ddp, opt, [0, 1, 2])
    pdt.utils.save_checkpoint(path, ddp, opt, epoch=3, extra={"note": "mid"})
    train(ddp, opt, [3, 4])
    want = torch.cat([p.detach().flatten() for p in ddp.parameters()])
    want_buf = ddp.module.layer1[1].running_mean.clone()

    ddp2, opt2 = fresh()
    if fuse:
        train(ddp2, opt2, [7, 8, 9])       # get the fused layout (flat momentum arena) in place before restoring into it
        assert opt2._fused_active
    info = pdt.utils.load_checkpoint(path, ddp2, opt2)
    assert info["epoch"] == 3 and info["extra"] == {"note": "mid"}
    train(ddp2, opt2, [3, 4])
    got = torch.cat([p.detach().flatten() for p in ddp2.parameters()])
    bare = pdt.models.ConvNet()
    pdt.utils.load_checkpoint(path, bare)  # module.-prefixed file into an unwrapped model
    same_buf = bool(torch.allclose(want_buf, ddp2.module.layer1[1].running_mean))
    return bool(torch.allclose(want, got, rtol=1e-6, atol=1e-7)), same_buf, os.path.exists(path)


@pytest.mark.parametrize("fuse", [False, True])
def test_checkpoint_resume_is_exact(tmp_path, fuse):
    res = run_ranks(_ckpt, 2, str(tmp_path / "ck.pt"), fuse)
    assert all(all(r) for r in res), res


def _logger(rank, world):
    ddp, _ = _train_ours(rank, world, 14)
    return ddp._get_ddp_logging_data()


def test_ddp_logging_data_running_averages():
    """B11: construction-time facts + runtime averages sampled after the first 10 iterations."""
    for d in run_ranks(_logger, 2):
        assert d["world_size"] == 2 and d["backend_name"] in ("gloo", "cpu") and d["num_parameter_tensors"] == 10
        assert d["bucket_sizes"] == [116136] and d["has_rebuilt_buckets"] and sorted(d["grad_ready_order"]) == list(range(10))
        assert d["num_iterations"] == 14 and d["timed_iterations"] == 4
        assert d["avg_forward_compute_time_us"] > 0 and d["avg_backward_compute_time_us"] > 0 and d["avg_backward_comm_time_us"] >= 0


def _powersgd(rank, world, rank_r):
    from pytorch_distributed_train_b200.parallel import comm_hooks

    torch.manual_seed(0)
    ddp = pdt.DistributedDataParallel(pdt.models.ConvNet())
    state = comm_hooks.PowerSGDState(matrix_approximation_rank=rank_r, start_powerSGD_iter=1, min_compression_rate=1.0)
    ddp.register_comm_hook(state, comm_hooks.powerSGD_hook)
    torch.manual_seed(0)
    plain = pdt.DistributedDataParallel(pdt.models.ConvNet())
    crit = nn.CrossEntropyLoss()
    errs = []
    for s in range(3):
        x, y = _data(rank, s)
        for m in (ddp, plain):
            m.zero_grad()
            crit(m(x), y).backward()
        a, b = ddp.module.fc.weight.grad, plain.module.fc.weight.grad
        errs.append(((a - b).norm() / b.norm()).item())
    return errs, ddp.module.fc.weight.grad.clone(), ddp.module.fc.bias.grad.clone(), plain.module.fc.bias.grad.clone(), len(state.errors)


def test_powersgd_hook_full_rank_is_exact_and_low_rank_agrees_across_ranks():
    full = run_ranks(_powersgd, 2, 10)   # fc.weight is 10×1568: rank 10 spans it
    for errs, _, bias, bias_ref, _ in full:
        assert errs[0] < 1e-5                       # first step uses the plain allreduce (start_powerSGD_iter=1)
        assert max(errs[1:]) < 1e-3, errs           # full-rank projection reproduces the averaged gradient
        assert torch.allclose(bias, bias_ref, atol=1e-6)  # 1-D tensors are never compressed
    low = run_ranks(_powersgd, 2, 1)
    assert torch.allclose(low[0][1], low[1][1], atol=1e-6), "every rank decompresses to the same gradient"
    assert 0.0 < max(low[0][0][1:]) < 1.0 and low[0][4] > 0   # lossy, with residuals kept for error feedback


def _unused_without_flag(rank, world):
    torch.manual_seed(0)
    ddp = pdt.DistributedDataParallel(_Branchy())       # find_unused_parameters=False (default)
    x = torch.randn(4, 4)
    ddp(x, False).sum().backward()                      # b and never produce no gradient: the bucket cannot complete
    try:
        ddp(x, False)
    except RuntimeError as e:
        return str(e)
    return ""


def test_unused_parameter_without_detection_is_diagnosed_not_silent():
    for msg in run_ranks(_unused_without_flag, 2):
        assert "Expected to have finished reduction in the prior iteration" in msg and "find_unused_parameters=True" in msg
