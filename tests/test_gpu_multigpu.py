"""Multi-GPU tests of the NVLink backend (SymmComm) against NCCL / closed-form results, and of DDP /
SyncBatchNorm end to end against the torch stack."""
import os

import pytest
import torch
import torch.nn as nn

import pytorch_distributed_train_b200 as pdt
from mp_helpers import free_port, run_ranks

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]
dist = pdt.distributed



def _world():
    return min(torch.cuda.device_count(), int(os.environ.get("PDT_TEST_WORLD", "8")))


def _collectives(rank, world):
    dev = torch.device("cuda", rank)
    comm = dist.get_default_group().comm
    info = {"desc": comm.describe(), "mc": comm.has_multicast}
    algos = ["oneshot", "twoshot"] + (["oneshot_mc", "nvls"] if comm.has_multicast else [])
    total = sum(range(1, world + 1))
    for algo in algos + ["auto"]:
        comm.algo = algo
        for n in (4, 1000, 29036, 262144, 1 << 20, (1 << 22) + 4):
            # symmetric (heap) buffer: zero-copy path
            t = comm.alloc_flat(n, torch.float32, dev)
            t.copy_(torch.arange(n, device=dev, dtype=torch.float32) % 97 * (rank + 1))
            dist.all_reduce(t)
            exp = torch.arange(n, device=dev, dtype=torch.float32) % 97 * total
            assert torch.equal(t, exp), f"{algo} heap n={n}"
            # ordinary tensor (staged path), odd length, averaged
            u = torch.full((n - 1,), float(rank + 1), device=dev)
            dist.all_reduce(u, dist.ReduceOp.AVG)
            assert torch.allclose(u, torch.full_like(u, total / world)), f"{algo} plain n={n - 1}"
            del t
    comm.algo = "auto"
    for dt in (torch.bfloat16, torch.float16, torch.float64, torch.int32, torch.int64):
        v = torch.ones(777, dtype=dt, device=dev) * (rank + 1)
        dist.all_reduce(v)
        assert torch.equal(v, torch.ones(777, dtype=dt, device=dev) * total), str(dt)
    m = torch.tensor([float(rank)], device=dev)
    dist.all_reduce(m, dist.ReduceOp.MAX)
    assert m.item() == world - 1
    # bitwise identical on every rank for random data, every algorithm
    sums = {}
    for algo in algos:
        comm.algo = algo
        g = torch.Generator(device=dev).manual_seed(rank)
        r = comm.alloc_flat(1 << 18, torch.float32, dev)
        r.copy_(torch.randn(1 << 18, device=dev, generator=g))
        dist.all_reduce(r)
        sums[algo] = r.view(torch.int32).sum().item()
    comm.algo = "auto"
    for root in range(world):
        b = torch.arange(1001, device=dev, dtype=torch.float32) + 7 * root if rank == root else torch.zeros(1001, device=dev)
        dist.broadcast(b, root)
        assert torch.equal(b, torch.arange(1001, device=dev, dtype=torch.float32) + 7 * root)
    nb = torch.zeros(3, dtype=torch.int64, device=dev) + (rank == 0) * 5
    dist.broadcast(nb, 0)
    assert nb.tolist() == [5, 5, 5]
    o = torch.empty(world * 5, device=dev)
    dist.all_gather_into_tensor(o, torch.full((5,), float(rank), device=dev))
    assert torch.equal(o, torch.arange(world, device=dev, dtype=torch.float32).repeat_interleave(5))
    a2a = torch.empty(world * 2, device=dev)
    dist.all_to_all_single(a2a, (torch.arange(world * 2, device=dev) // 2 + 10 * rank).float())
    assert torch.equal(a2a, torch.tensor([10.0 * r + rank for r in range(world) for _ in range(2)], device=dev))
    dist.barrier()
    torch.cuda.synchronize()
    info["sums"] = sums
    info["status"] = comm.status()
    return info


def test_symm_collectives():
    w = _world()
    res = run_ranks(_collectives, w, backend="nccl")
    for algo in res[0]["sums"]:
        assert len({r["sums"][algo] for r in res}) == 1, f"{algo}: results differ between ranks"
    assert all(r["status"] == 0 for r in res)
    print(res[0]["desc"])


def _vs_nccl(rank, world):
    """Same inputs through SymmComm and through the libnccl binding."""
    dev = torch.device("cuda", rank)
    g = dist.get_default_group()
    ref = dist.new_group(comm="nccl")
    gen = torch.Generator(device=dev).manual_seed(100 + rank)
    out = []
    for n in (29034, 1 << 16, 3_000_001):
        x = torch.randn(n, device=dev, generator=gen)
        a, b = x.clone(), x.clone()
        dist.all_reduce(a, group=g)
        dist.all_reduce(b, group=ref)
        out.append((a - b).abs().max().item() / (b.abs().max().item() + 1e-9))
    return out


def test_allreduce_matches_nccl():
    for errs in run_ranks(_vs_nccl, _world(), backend="nccl"):
        assert max(errs) < 1e-5, errs


def _data(rank, step, bs=100):
    g = torch.Generator().manual_seed(1000 * step + rank)
    return torch.rand(bs, 1, 28, 28, generator=g), torch.randint(0, 10, (bs,), generator=g)


def _ddp_vs_torch(rank, world, syncbn, port):
    import torch.distributed as td

    dev = torch.device("cuda", rank)
    torch.backends.cudnn.allow_tf32 = False
    steps = 4
    torch.manual_seed(0)
    model = pdt.models.ConvNet()
    if syncbn:
        model = pdt.SyncBatchNorm.convert_sync_batchnorm(model)
    model.to(dev)
    opt = pdt.optim.SGD(model.parameters(), 0.01)  # (0.05 makes the loss climb 2.4 → 13: rounding noise gets amplified)
    ddp = pdt.DistributedDataParallel(model, device_ids=[rank])
    crit = pdt.nn.CrossEntropyLoss()
    ours = []
    for s in range(steps):
        x, y = _data(rank, s)
        loss = crit(ddp(x.to(dev)), y.to(dev))
        opt.zero_grad()
        loss.backward()
        opt.step()
        ours.append(loss.item())
    info = ddp._get_ddp_logging_data()
    td.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", world_size=world, rank=rank)
    torch.manual_seed(0)
    ref = pdt.models.ConvNet(fused=False)
    if syncbn:
        ref = nn.SyncBatchNorm.convert_sync_batchnorm(ref)
    ref.to(dev)
    ropt = torch.optim.SGD(ref.parameters(), 0.01)
    rddp = nn.parallel.DistributedDataParallel(ref, device_ids=[rank])
    theirs = []
    for s in range(steps):
        x, y = _data(rank, s)
        loss = nn.functional.cross_entropy(rddp(x.to(dev)), y.to(dev))
        ropt.zero_grad()
        loss.backward()
        ropt.step()
        theirs.append(loss.item())
    worst = 0.0
    for (n, p), (_, q) in zip(ddp.module.named_parameters(), rddp.module.named_parameters()):
        worst = max(worst, (p - q).abs().max().item() / (q.abs().max().item() + 1e-6))
    bufw = 0.0
    for (n, p), (_, q) in zip(ddp.module.named_buffers(), rddp.module.named_buffers()):
        bufw = max(bufw, (p.float() - q.float()).abs().max().item())
    flat = torch.cat([p.detach().reshape(-1) for p in ddp.parameters()])
    td.destroy_process_group()
    return {"ours": ours, "theirs": theirs, "param_rel": worst, "buf_abs": bufw, "psum": flat.double().sum().item(),
            "copies": info["copies_into_bucket"], "buckets": info["bucket_sizes"]}


@pytest.mark.parametrize("syncbn", [False, True])
def test_ddp_convnet_matches_torch_ddp_nccl(syncbn):
    res = run_ranks(_ddp_vs_torch, _world(), syncbn, free_port(), backend="nccl")
    assert len({r["psum"] for r in res}) == 1, "parameters diverged between ranks"
    for r in res:
        assert max(abs(a - b) for a, b in zip(r["ours"], r["theirs"])) < 5e-3, (r["ours"], r["theirs"])
        # conv weight gradients behind a BatchNorm are ill-conditioned: TF32 (ours) vs fp32 cuDNN differ by up to
        # 3.7e-2 of the max entry, the same as cuDNN-TF32 vs float64
        assert r["param_rel"] < 5e-2 and r["buf_abs"] < 5e-3, r
        assert r["copies"] == 0 and sum(r["buckets"]) == 116136


def _resnet(rank, world, syncbn, port):
    """BASELINE.json config 4 at test scale: multi-bucket reduce (11.7 M params) + generic SyncBN kernels."""
    import torch.distributed as td

    dev = torch.device("cuda", rank)
    steps = 3
    # fp32 convolutions in both arms: with TF32 operand rounding a 1e-7 difference between our SyncBN arithmetic (fp64 sums) and
    # torch's (Welford) flips roundings in the next convolution, and layer4's BatchNorm over 4·2·2·world samples amplifies that to
    # several percent of the gradient — a property of the comparison, not of either implementation
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False

    def data(s):
        # seeds 77·(s+1)+rank: the batch of tools/numerics_probe.py.  With seed = rank the same comparison is off by up to 20 % in
        # layer4 for OUR kernels and for our torch-op fallback math alike: 8 samples
        # per rank reach layer4's BatchNorm at 2×2 resolution, and channels that are (almost) constant after the ReLU get
        # invstd = 1/sqrt(eps) = 316 — two correct ways of summing (fp64 Σx, Σx² here, Welford in torch) then disagree visibly.
        g = torch.Generator().manual_seed(77 * (s + 1) + rank)
        return torch.randn(4, 3, 64, 64, generator=g).to(dev), torch.randint(0, 10, (4,), generator=g).to(dev)

    torch.manual_seed(0)
    net = pdt.models.resnet18(num_classes=10)
    if syncbn:
        net = pdt.SyncBatchNorm.convert_sync_batchnorm(net)
    net.to(dev)
    watch = ("conv1.weight", "bn1.weight", "layer2.0.bn2.bias", "layer4.1.bn2.weight", "fc.weight")
    opt = pdt.optim.SGD(net.parameters(), 0.01, momentum=0.9)
    ddp = pdt.DistributedDataParallel(net, device_ids=[rank], bucket_cap_mb=8, first_bucket_cap_mb=1)
    ours, g_ours = [], {}
    for s in range(steps):
        x, y = data(s)
        loss = nn.functional.cross_entropy(ddp(x), y)
        opt.zero_grad()
        loss.backward()
        if s == 0:
            g_ours = {n: p.grad.detach().clone() for n, p in ddp.module.named_parameters() if n in watch}
        opt.step()
        ours.append(loss.item())
    info = ddp._get_ddp_logging_data()
    td.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", world_size=world, rank=rank)
    torch.manual_seed(0)
    ref = pdt.models.resnet18(num_classes=10)
    if syncbn:
        ref = nn.SyncBatchNorm.convert_sync_batchnorm(ref)
    ref.to(dev)
    ropt = torch.optim.SGD(ref.parameters(), 0.01, momentum=0.9)
    rddp = nn.parallel.DistributedDataParallel(ref, device_ids=[rank], bucket_cap_mb=8)
    theirs, grad_rel = [], {}
    for s in range(steps):
        x, y = data(s)
        loss = nn.functional.cross_entropy(rddp(x), y)
        ropt.zero_grad()
        loss.backward()
        if s == 0:  # first-step averaged gradients: same weights, same data -> must agree to TF32 rounding
            for n, p in rddp.module.named_parameters():
                if n in watch:
                    grad_rel[n] = ((p.grad - g_ours[n]).abs().max() / (p.grad.abs().max() + 1e-12)).item()
        ropt.step()
        theirs.append(loss.item())
    td.destroy_process_group()
    flat = torch.cat([p.detach().reshape(-1) for p in ddp.parameters()])
    return {"ours": ours, "theirs": theirs, "psum": flat.double().sum().item(), "buckets": info["bucket_sizes"], "grad_rel": grad_rel}


@pytest.mark.parametrize("syncbn", [False, True])
def test_ddp_resnet18_multibucket_matches_torch(syncbn):
    # Two ranks whatever the box has: the comparison is about multi-bucket / chunked reduction order and the generic SyncBN
    # kernels, which do not depend on the world size, while its conditioning does (the 4-image batch per rank and the seeds were
    # picked and validated for two ranks, see _resnet.data); collectives at the full world size are covered by the tests above.
    res = run_ranks(_resnet, min(_world(), 2), syncbn, free_port(), backend="nccl")
    assert len({r["psum"] for r in res}) == 1, "parameters diverged between ranks"
    assert len(res[0]["buckets"]) >= 3 and sum(res[0]["buckets"]) == 4 * 11181642
    for r in res:
        assert max(r["grad_rel"].values()) < 1e-3, r["grad_rel"]
        assert max(abs(a - b) for a, b in zip(r["ours"], r["theirs"])) < 5e-3, (r["ours"], r["theirs"], r["grad_rel"])


def _graphed(rank, world, syncbn):
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    dev = torch.device("cuda", rank)
    torch.manual_seed(0)
    model = pdt.models.ConvNet()
    if syncbn:
        model = pdt.SyncBatchNorm.convert_sync_batchnorm(model)
    model.to(dev)
    opt = pdt.optim.SGD(model.parameters(), 0.05)
    ddp = pdt.DistributedDataParallel(model, device_ids=[rank])
    crit = pdt.nn.CrossEntropyLoss()
    x, y = _data(rank, 0)
    step = GraphedTrainStep(ddp, crit, opt, (x.to(dev), y.to(dev)))
    losses = []
    for s in range(50):
        x, y = _data(rank, s % 5)
        losses.append(step(x.pin_memory(), y.pin_memory()).item())
    flat = torch.cat([p.detach().reshape(-1) for p in ddp.parameters()])
    return losses[0], losses[-1], flat.double().sum().item(), step.kernels_per_replay


@pytest.mark.parametrize("syncbn", [False, True])
def test_graph_captured_step_keeps_ranks_in_lockstep(syncbn):
    res = run_ranks(_graphed, _world(), syncbn, backend="nccl")
    assert len({r[2] for r in res}) == 1
    assert all(r[1] < r[0] for r in res), res
    print("kernels per replay:", res[0][3])


def _fused_sgd(rank, world, momentum):
    """One-kernel allreduce+SGD (optim.SGD.fuse_with_ddp) vs the reducer-driven two-kernel path, eager
    and graph-captured: same parameters after the same steps."""
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    dev = torch.device("cuda", rank)
    outs = []
    for mode in ("plain", "fused", "fused_graph"):
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(dev)
        opt = pdt.optim.SGD(model.parameters(), 0.01, momentum=momentum, weight_decay=1e-3 if momentum else 0.0)
        ddp = pdt.DistributedDataParallel(model, device_ids=[rank])
        crit = pdt.nn.CrossEntropyLoss()
        if mode == "fused_graph":
            x, y = _data(rank, 0)
            step = GraphedTrainStep(ddp, crit, opt, (x.to(dev), y.to(dev)), warmup=0)
            assert step.fused_optimizer
            # the capture ran max(warmup, 4) eager steps on batch 0: redo the same on the other arms
            for s in range(8):
                x, y = _data(rank, s)
                step(x.pin_memory(), y.pin_memory())
        else:
            if mode == "fused":
                opt.fuse_with_ddp(ddp)
            for s in [0, 0, 0, 0] + list(range(8)):
                x, y = _data(rank, s)
                loss = crit(ddp(x.to(dev)), y.to(dev))
                opt.zero_grad()
                loss.backward()
                opt.step()
            assert bool(opt._fused_active) == (mode == "fused")
        torch.cuda.synchronize()
        outs.append(torch.cat([p.detach().reshape(-1) for p in ddp.parameters()]).cpu())
    return outs


@pytest.mark.parametrize("momentum", [0.0, 0.9])
def test_fused_allreduce_sgd(momentum):
    res = run_ranks(_fused_sgd, _world(), momentum, backend="nccl")
    for plain, fused, graphed in res:
        # the two paths differ by FMA ordering only (1 ulp), but TF32 operand rounding inside the
        # convolutions turns a 1-ulp weight change into an up-to-2^-11 effective change: compare at that floor
        scale = plain.abs().max().item()
        assert (plain - fused).abs().max().item() < 2e-3 * scale, ((plain - fused).abs().max(), scale)
        assert (plain - graphed).abs().max().item() < 2e-3 * scale, ((plain - graphed).abs().max(), scale)
    assert torch.equal(res[0][1], res[-1][1]) and torch.equal(res[0][2], res[-1][2])  # ranks bit-identical


def _rooted(rank, world):
    """reduce / reduce_scatter / gather / scatter: one barrier-synchronised kernel over the staging area each."""
    dev = torch.device("cuda", rank)
    total = sum(range(1, world + 1))
    for n in (5, 1000, 262147):
        for root in (0, world - 1):
            t = torch.arange(n, device=dev, dtype=torch.float32) % 13 * (rank + 1)
            dist.reduce(t, root)
            if rank == root:
                assert torch.equal(t, torch.arange(n, device=dev, dtype=torch.float32) % 13 * total), ("reduce", n, root)
            g = torch.full((n,), float(rank), device=dev)
            outs = [torch.empty(n, device=dev) for _ in range(world)] if rank == root else None
            dist.gather(g, outs, dst=root)
            if rank == root:
                assert all(torch.equal(o, torch.full((n,), float(r), device=dev)) for r, o in enumerate(outs)), ("gather", n, root)
            sc = torch.empty(n, device=dev)
            dist.scatter(sc, [torch.full((n,), float(10 * r + root), device=dev) for r in range(world)] if rank == root else None, src=root)
            assert torch.equal(sc, torch.full((n,), float(10 * rank + root), device=dev)), ("scatter", n, root)
        inp = (torch.arange(world * n, device=dev, dtype=torch.float32) % 7 + rank).contiguous()
        out = torch.empty(n, device=dev)
        dist.reduce_scatter_tensor(out, inp)
        exp = (torch.arange(world * n, device=dev, dtype=torch.float32) % 7)[rank * n:(rank + 1) * n] * world + sum(range(world))
        assert torch.equal(out, exp), ("reduce_scatter", n)
    mx = torch.tensor([float(rank)], device=dev)
    dist.reduce(mx, 0, dist.ReduceOp.MAX)
    assert rank != 0 or mx.item() == world - 1
    torch.cuda.synchronize()
    return True


def test_rooted_collectives_over_the_symmetric_heap():
    assert all(run_ranks(_rooted, _world(), backend="nccl"))


def _absent_rank(rank, world, init, outdir):
    import json
    import time

    os.environ["PDT_SYMM_TIMEOUT_S"] = "3"
    torch.cuda.set_device(rank)
    pdt.init_process_group("nccl", init_method=init, world_size=world, rank=rank, timeout=60.0)
    comm = dist.get_default_group().comm
    t = torch.ones(1024, device=f"cuda:{rank}")
    dist.all_reduce(t)
    torch.cuda.synchronize()  # a healthy collective first
    msg, t0 = "none", time.time()
    if rank != world - 1:
        try:
            dist.all_reduce(t)  # the last rank never joins this one
            torch.cuda.synchronize()
        except Exception as e:  # the kernel's globaltimer watchdog trapped
            msg = f"{type(e).__name__}: {e}"
    else:
        time.sleep(8.0)
    with open(os.path.join(outdir, f"r{rank}.json"), "w") as f:
        json.dump({"msg": msg[:200], "status": comm.status(), "text": comm.status_string(), "seconds": time.time() - t0}, f)
        f.flush()
    os._exit(0)  # the CUDA context of the timed-out ranks is gone: skip orderly teardown


def test_absent_rank_trips_the_device_side_timeout(tmp_path):
    """A rank that never joins a collective must produce a diagnostic within the
    configured timeout on every waiting rank, not a hang."""
    import json

    w = _world()
    pdt.spawn(_absent_rank, args=(w, f"tcp://127.0.0.1:{free_port()}", str(tmp_path)), nprocs=w, grace_period=5.0)
    res = [json.load(open(tmp_path / f"r{r}.json")) for r in range(w)]
    for r in range(w - 1):
        assert res[r]["status"] != 0 and f"never heard from rank {w - 1}" in res[r]["text"], res[r]
        assert res[r]["msg"] != "none" and res[r]["seconds"] < 30
    assert res[w - 1]["status"] == 0


def _stress(rank, world):
    """Stress: 10k back-to-back collectives with randomised per-rank stream delays — the
    flag/epoch protocol must neither deadlock nor let a fast rank overwrite a slot a slow rank is reading."""
    import random

    dev = torch.device("cuda", rank)
    comm = dist.get_default_group().comm
    rng = random.Random(1234 + rank)
    small = torch.zeros(257, device=dev)          # odd length: vector body + tail
    heap = comm.alloc_flat(4096, torch.float32, dev)
    expect_small = expect_heap = 0.0
    total = sum(range(1, world + 1))
    for i in range(10000):
        if rng.random() < 0.02:
            torch.cuda._sleep(rng.randrange(20000, 400000))   # 10–200 µs of stall on this rank only
        small.fill_(float(rank + 1))
        comm.allreduce_inline(small, dist.ReduceOp.SUM, 1.0)
        if i % 7 == 0:
            heap.fill_(float(rank + 1) * (i % 5))
            comm.allreduce(heap, dist.ReduceOp.SUM, 1.0).wait()   # comm-stream channel interleaved with the inline one
            expect_heap = float(total * (i % 5))
        if i % 1000 == 999:
            assert small.eq(float(total)).all().item(), i
            assert heap.eq(expect_heap).all().item(), i
    torch.cuda.synchronize()
    return comm.status()


def test_ten_thousand_back_to_back_collectives():
    assert run_ranks(_stress, _world(), backend="nccl") == [0] * _world()


def _p2p(rank, world):
    """send / recv over the symmetric heap: ring exchange (eager, so send-then-recv does not deadlock), a message larger
    than one staging half (chunked, needs the matching recv posted), an empty tensor."""
    dev = torch.device("cuda", rank)
    nxt, prv = (rank + 1) % world, (rank - 1) % world
    out = torch.full((1000,), float(rank), device=dev)
    inp = torch.empty(1000, device=dev)
    dist.send(out, nxt)
    dist.recv(inp, prv)
    ok = bool(inp.eq(float(prv)).all())
    big = 5 * (1 << 20) + 3                                   # 20 MB + 12 B of fp32: two chunks
    if rank == 0:
        dist.send(torch.arange(big, device=dev, dtype=torch.float32), 1)
        dist.send(torch.empty(0, device=dev), 1)
    elif rank == 1:
        got = torch.empty(big, device=dev)
        dist.recv(got, 0)
        ok = ok and bool(torch.equal(got, torch.arange(big, device=dev, dtype=torch.float32)))
        dist.recv(torch.empty(0, device=dev), 0)
    dist.barrier()
    return ok


def test_send_recv_over_the_symmetric_heap():
    assert all(run_ranks(_p2p, _world(), backend="nccl"))
