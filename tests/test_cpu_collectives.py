"""CPU backend collectives over our TCP mesh, world sizes 2-4 (BASELINE.json config 1 plumbing)."""
import pytest
import torch

import pytorch_distributed_train_b200 as pdt
from mp_helpers import run_ranks

dist = pdt.distributed


def _collectives(rank, world):
    out = {}
    # allreduce small / large(ring) / odd sizes / dtypes
    for n in (1, 7, 1000, 100003):
        t = torch.arange(n, dtype=torch.float32) * (rank + 1)
        dist.all_reduce(t)
        exp = torch.arange(n, dtype=torch.float32) * sum(r + 1 for r in range(world))
        assert torch.equal(t, exp), f"allreduce n={n}"
    t = torch.full((5,), float(rank))
    dist.all_reduce(t, dist.ReduceOp.MAX)
    assert torch.equal(t, torch.full((5,), float(world - 1)))
    t = torch.full((5,), float(rank + 1))
    dist.all_reduce(t, dist.ReduceOp.AVG)
    assert torch.allclose(t, torch.full((5,), sum(range(1, world + 1)) / world))
    for dt in (torch.int64, torch.int32, torch.float64, torch.bfloat16, torch.float16, torch.uint8):
        t = torch.ones(33, dtype=dt) * (rank + 1)
        dist.all_reduce(t)
        assert torch.equal(t, torch.ones(33, dtype=dt) * sum(range(1, world + 1))), str(dt)
    # bitwise identical results on all ranks for a big random vector (ring path)
    g = torch.Generator().manual_seed(rank)
    big = torch.randn(300000, generator=g)
    dist.all_reduce(big)
    out["big_sum_bits"] = big.view(torch.int32).sum().item()
    # broadcast from every root
    for root in range(world):
        t = torch.arange(10.0) + 100 * root if rank == root else torch.zeros(10)
        dist.broadcast(t, root)
        assert torch.equal(t, torch.arange(10.0) + 100 * root)
    # allgather
    o = torch.empty(world * 3)
    dist.all_gather_into_tensor(o, torch.full((3,), float(rank)))
    assert torch.equal(o, torch.arange(world, dtype=torch.float32).repeat_interleave(3))
    lst = [torch.empty(2) for _ in range(world)]
    dist.all_gather(lst, torch.full((2,), float(rank)))
    assert all(torch.equal(lst[r], torch.full((2,), float(r))) for r in range(world))
    # reduce / reduce_scatter / gather / scatter / alltoall / send-recv
    t = torch.ones(4) * (rank + 1)
    dist.reduce(t, 0)
    if rank == 0:
        assert torch.equal(t, torch.ones(4) * sum(range(1, world + 1)))
    rs = torch.empty(2)
    dist.reduce_scatter_tensor(rs, torch.arange(2.0 * world) + rank)
    assert torch.equal(rs, (torch.arange(2.0 * world) * world + sum(range(world)))[2 * rank:2 * rank + 2])
    gl = [torch.empty(1) for _ in range(world)] if rank == 1 else None
    dist.gather(torch.tensor([float(rank)]), gl, dst=1)
    if rank == 1:
        assert [int(x.item()) for x in gl] == list(range(world))
    sc = torch.empty(2)
    dist.scatter(sc, [torch.full((2,), float(r)) for r in range(world)] if rank == 0 else None, src=0)
    assert torch.equal(sc, torch.full((2,), float(rank)))
    a2a = torch.empty(world)
    dist.all_to_all_single(a2a, torch.arange(world, dtype=torch.float32) + 10 * rank)
    assert torch.equal(a2a, torch.tensor([10.0 * r + rank for r in range(world)]))
    if rank == 0:
        dist.send(torch.tensor([42.0]), 1)
    elif rank == 1:
        r = torch.empty(1)
        dist.recv(r, 0)
        assert r.item() == 42.0
    dist.barrier()
    w = dist.all_reduce(torch.ones(3), async_op=True)
    assert w.wait() is True
    objs = dist.all_gather_object({"r": rank})
    assert [o["r"] for o in objs] == list(range(world))
    assert dist.broadcast_object("hello" if rank == 0 else None, 0) == "hello"
    out["rank"], out["world"], out["backend"] = dist.get_rank(), dist.get_world_size(), dist.get_backend()
    out["records"] = len(dist.get_default_group().comm.flight_records())
    return out


@pytest.mark.parametrize("world", [2, 3, 4])
def test_collectives(world):
    res = run_ranks(_collectives, world)
    assert [r["rank"] for r in res] == list(range(world))
    assert all(r["world"] == world and r["backend"] == "gloo" for r in res)
    assert len({r["big_sum_bits"] for r in res}) == 1, "allreduce must be bitwise identical across ranks"
    assert all(r["records"] > 0 for r in res)


def _subgroups(rank, world):
    g = dist.new_group([0, 2])
    t = torch.ones(2) * (rank + 1)
    if g is not None:
        dist.all_reduce(t, group=g)
        assert torch.equal(t, torch.ones(2) * 4) and g.size() == 2
    else:
        assert rank == 1
    dist.monitored_barrier()
    return True


def test_new_group():
    assert all(run_ranks(_subgroups, 3))


def _double_init(rank, world):
    try:
        pdt.init_process_group("gloo", init_method="tcp://127.0.0.1:1", world_size=1, rank=0)
    except RuntimeError as e:
        return "twice" in str(e)
    return False


def test_double_init_is_an_error():
    assert all(run_ranks(_double_init, 2))


def _dead_peer(rank, world):
    import os
    import time

    if rank == 1:
        os._exit(7)  # dies before joining the collective
    t = torch.ones(4)
    t0 = time.time()
    try:
        dist.all_reduce(t)
    except Exception as e:  # PeerClosedError / TimeoutError
        return ("err", type(e).__name__, time.time() - t0)
    return ("no-error",)


def test_dead_rank_fails_fast_instead_of_hanging():
    from pytorch_distributed_train_b200 import launcher

    with pytest.raises((launcher.ProcessExitedException, launcher.ProcessRaisedException)):
        run_ranks(_dead_peer, 2, grace_period=2.0)


def test_single_process_env_rendezvous(monkeypatch):
    from mp_helpers import free_port

    monkeypatch.setenv("MASTER_ADDR", "127.0.0.1")
    monkeypatch.setenv("MASTER_PORT", str(free_port()))
    monkeypatch.setenv("RANK", "0")
    monkeypatch.setenv("WORLD_SIZE", "1")
    pdt.init_process_group("gloo")
    try:
        t = torch.ones(3)
        dist.all_reduce(t)
        assert torch.equal(t, torch.ones(3)) and dist.get_world_size() == 1
    finally:
        pdt.destroy_process_group()
    assert not dist.is_initialized()


def test_file_rendezvous(tmp_path):
    pdt.init_process_group("gloo", init_method=f"file://{tmp_path}/rdzv", world_size=1, rank=0)
    pdt.destroy_process_group()


def _debug_detail(rank, world):
    import os

    os.environ["PDT_DISTRIBUTED_DEBUG"] = "DETAIL"
    t = torch.ones(4)
    dist.all_reduce(t)  # matching call passes the fingerprint check
    assert t[0].item() == world
    try:
        if rank == 0:
            dist.all_reduce(torch.ones(4))
        else:
            dist.broadcast(torch.ones(5), 0)  # wrong collective, wrong shape
    except RuntimeError as e:
        msg = str(e)
    else:
        msg = ""
    os.environ["PDT_DISTRIBUTED_DEBUG"] = "OFF"
    os.environ["PDT_NAN_CHECK"] = "1"
    try:
        dist.all_reduce(torch.tensor([1.0, float("nan")]))
    except RuntimeError as e:
        nan_msg = str(e)
    else:
        nan_msg = ""
    os.environ["PDT_NAN_CHECK"] = "0"
    return msg, nan_msg


def test_debug_detail_names_mismatched_collectives_and_nan_check():
    """Collective fingerprint check + NaN check instead of a hang / silent corruption."""
    for msg, nan_msg in run_ranks(_debug_detail, 2):
        assert "collective mismatch at sequence number 2" in msg and "all_reduce" in msg and "broadcast" in msg
        assert "non-finite" in nan_msg


def _object_collectives(rank, world):
    store = dist.get_store()
    before = store.num_keys()
    objs = [{"a": 1}, "x", 3.5] if rank == 1 else [None, None, None]
    dist.broadcast_object_list(objs, src=1)
    gathered = [None] * world if rank == 0 else None
    dist.gather_object(("r", rank), gathered, dst=0)
    out = [None]
    dist.scatter_object_list(out, [f"for-{r}" for r in range(world)] if rank == 0 else None, src=0)
    b = dist.broadcast_object({"k": [1, 2]} if rank == 0 else None, 0)
    dist.barrier()
    return objs, gathered, out[0], b, store.num_keys() - before


def test_object_collectives_and_store_hygiene():
    res = run_ranks(_object_collectives, 2)
    for rank, (objs, gathered, got, b, grown) in enumerate(res):
        assert objs == [{"a": 1}, "x", 3.5] and got == f"for-{rank}" and b == {"k": [1, 2]}
        assert gathered == ([("r", 0), ("r", 1)] if rank == 0 else None)
        assert grown <= 2, "object exchanges must clean their keys out of the store"


def _list_forms_and_p2p_batches(rank, world):
    # all_to_all (list form): input j goes to rank j
    outs = [torch.empty(3) for _ in range(world)]
    dist.all_to_all(outs, [torch.full((3,), float(10 * rank + j)) for j in range(world)])
    assert all(torch.equal(outs[i], torch.full((3,), float(10 * i + rank))) for i in range(world))
    w = dist.all_to_all(outs, [torch.full((3,), float(100 * rank + j)) for j in range(world)], async_op=True)
    assert w.wait() and w.is_completed()
    assert all(torch.equal(outs[i], torch.full((3,), float(100 * i + rank))) for i in range(world))
    # reduce_scatter (list form): rank i gets Σ_r input_list[i] of rank r
    o = torch.empty(2)
    dist.reduce_scatter(o, [torch.full((2,), float(rank + 1) * (j + 1)) for j in range(world)])
    assert torch.equal(o, torch.full((2,), float(sum(range(1, world + 1)) * (rank + 1))))
    # rank translation on a sub-group with non-trivial ranks
    g = dist.new_group([1, 2])
    assert dist.get_process_group_ranks() == list(range(world)) and dist.get_global_rank(None, 1) == 1
    if g is not None:
        assert dist.get_process_group_ranks(g) == [1, 2]
        assert dist.get_group_rank(g, 2) == 1 and dist.get_global_rank(g, 0) == 1
        try:
            dist.get_group_rank(g, 0)
            raise AssertionError("rank 0 is not in the group")
        except ValueError:
            pass
    # a ring exchange as one batch of point-to-point operations: everybody sends right and receives from the left
    right, left = (rank + 1) % world, (rank - 1) % world
    got = torch.empty(4)
    works = dist.batch_isend_irecv([dist.P2POp(dist.isend, torch.full((4,), float(rank)), right), dist.P2POp(dist.irecv, got, left)])
    for wk in works:
        wk.wait()
    assert torch.equal(got, torch.full((4,), float(left)))
    try:
        dist.P2POp(dist.send, got, left)
        raise AssertionError("only isend / irecv are valid batch members")
    except ValueError:
        pass
    dist.barrier()
    return True


def test_list_collectives_rank_translation_and_p2p_batches():
    assert all(run_ranks(_list_forms_and_p2p_batches, 3))
