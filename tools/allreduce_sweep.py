#!/usr/bin/env python
"""Allreduce latency / bus-bandwidth sweep: our NVLink kernels vs the libnccl baseline
(BASELINE.json config 5: "allreduce bus-bandwidth sweep 1KB–1GB at 2/4/8 GPUs vs reference NCCL").

    python tools/allreduce_sweep.py --gpus 8 [--max-mb 256] [--out sweep_8.json]

Every number is device-timed with CUDA events on the launching stream, after warm-up, with a
barrier + synchronize on both sides, and is the MAX over ranks.  busbw = 2(N-1)/N · bytes / t.
Roofline: t_min = bytes_that_must_cross_NVLink / 450 GB/s per direction per GPU (H100 SXM, NVLink 4 data sheet);
one-shot push sends (N-1)·S, NVLS two-shot moves ≈ S in + S out per GPU, P2P two-shot 2·S·(N-1)/N.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LINK_GBS = 450.0


def roofline_us(algo, nbytes, n):
    if algo in ("oneshot", "oneshot_mc"):
        cross = nbytes * (n - 1) if algo == "oneshot" else nbytes
    elif algo == "nvls":
        cross = nbytes  # S/N reduced in + (N-1)S/N broadcast in per GPU ≈ S
    else:
        cross = 2 * nbytes * (n - 1) / n
    return cross / (LINK_GBS * 1e3)


def worker(rank, world, max_mb, iters, out_path):
    import torch

    import pytorch_distributed_train_b200 as pdt

    dist = pdt.distributed
    dev = torch.device("cuda", rank)
    g = dist.get_default_group()
    comm = g.comm
    ref = dist.new_group(comm="nccl")
    algos = ["oneshot", "twoshot"] + (["oneshot_mc", "nvls"] if comm.has_multicast else [])
    sizes = []
    s = 1024
    while s <= max_mb << 20:
        sizes.append(s)
        s *= 4
    sizes.insert(4, 116136 // 16 * 16 + 16)  # the ConvNet bucket
    rows = []

    def timeit(fn, n_iter):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        dist.barrier()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n_iter):
            fn()
        b.record()
        torch.cuda.synchronize()
        t = torch.tensor([a.elapsed_time(b) / n_iter * 1e3], device=dev)  # us
        dist.all_reduce(t, dist.ReduceOp.MAX)
        return float(t.item())

    for nbytes in sizes:
        n = nbytes // 4
        buf = comm.alloc_flat(n, torch.float32, dev)
        buf.fill_(1.0)
        plain = torch.ones(n, device=dev)
        n_iter = max(5, min(iters, int(2e9 / max(nbytes, 1 << 16))))
        row = {"bytes": nbytes}

        def run_nccl():
            ref.comm.allreduce(plain, dist.ReduceOp.SUM, 1.0).wait()

        row["nccl_us"] = timeit(run_nccl, n_iter)
        for algo in algos:
            if algo.startswith("oneshot") and nbytes * world > (16 << 20):
                continue
            comm.algo = algo

            def run():
                comm.allreduce(buf, dist.ReduceOp.SUM, 1.0).wait()

            try:
                row[algo + "_us"] = timeit(run, n_iter)
            except Exception as e:  # noqa: BLE001
                row[algo + "_err"] = str(e)[:100]
        comm.algo = "auto"

        def run_auto():
            comm.allreduce(buf, dist.ReduceOp.SUM, 1.0).wait()

        row["auto_us"] = timeit(run_auto, n_iter)

        # Device-side latency without host launch/stream-hop overhead: 16 back-to-back collectives
        # captured in one CUDA graph (how they run inside the graph-replayed training step).
        def graphed(fn):
            chain = 16
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                fn()
            torch.cuda.current_stream(dev).wait_stream(side)
            torch.cuda.synchronize()
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, stream=side):
                for _ in range(chain):
                    fn()
            return timeit(gr.replay, max(5, n_iter // chain)) / chain

        if nbytes <= (4 << 20):
            try:
                row["graph_ours_us"] = graphed(lambda: comm.allreduce_inline(buf, dist.ReduceOp.SUM, 1.0))
                row["graph_nccl_us"] = graphed(lambda: ref.comm.allreduce(plain, dist.ReduceOp.SUM, 1.0).wait())
            except Exception as e:  # noqa: BLE001
                row["graph_err"] = str(e)[:120]
        best = min((v, k) for k, v in row.items() if k.endswith("_us") and not k.startswith("nccl") and k != "auto_us")
        row["best"] = best[1][:-3]
        row["best_us"] = best[0]
        row["busbw_gbs"] = 2 * (world - 1) / world * nbytes / (best[0] * 1e-6) / 1e9
        row["nccl_busbw_gbs"] = 2 * (world - 1) / world * nbytes / (row["nccl_us"] * 1e-6) / 1e9
        row["roofline_us"] = roofline_us(row["best"], nbytes, world)
        row["roofline_frac"] = row["roofline_us"] / best[0]
        row["speedup_vs_nccl"] = row["nccl_us"] / best[0]
        rows.append(row)
        del buf
        if rank == 0:
            print(json.dumps(row), flush=True)
    if rank == 0 and out_path:
        with open(out_path, "w") as f:
            json.dump({"world": world, "link_gbs": LINK_GBS, "desc": comm.describe(), "rows": rows}, f, indent=1)
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=2)
    ap.add_argument("--max-mb", type=int, default=256)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from mp_helpers import run_ranks

    os.environ.setdefault("PDT_SYMM_HEAP_MB", str(max(1024, 3 * a.max_mb + 128)))
    run_ranks(worker, a.gpus, a.max_mb, a.iters, a.out, backend="nccl")


if __name__ == "__main__":
    main()
