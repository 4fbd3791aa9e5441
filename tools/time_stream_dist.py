#!/usr/bin/env python3
"""A job whose ranks stream their own shares of bench.py's workload (BASELINE.json configs[1]) under a device budget
(dist.StreamedShardedScan, DESIGN.md §4c, *Ranks*), next to the in-process streamed call on the same table: per rank
and per scan, the chunk loop (pass 1), the verdict and S index, the Bloom all-gather, and per exchange round the
resolve, the query all-to-all, the answers, the answer all-to-all and the settle; rounds, queries per owner and
device bytes.  Prints one JSON line on rank 0; exits 3 unless every plot equals the in-process streamed plot.
Writes nothing to the tree.

    torchrun --nproc-per-node W tools/time_stream_dist.py --budget-gb 1.6 [--nels 2e8] [--steps 3] [--warmup 1]

Several ranks run NCCL when there is a GPU per rank, else gloo with every rank on GPU 0 (then the budget is per
rank and the ranks share the card).
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import COV, HET, K, LCUT, PLOIDY, SEED, workload_name  # noqa: E402
from smudgeplot_b200 import _lib  # noqa: E402
from tools import synth  # noqa: E402
from tools.time_stream import host_records, power_limit  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--budget-gb", type=float, required=True, help="device budget of each rank (GB)")
    ap.add_argument("--nels", type=float, default=2e8)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    import torch
    import torch.distributed as dist
    from smudgeplot_b200 import dist as hd
    if not torch.cuda.is_available():
        raise SystemExit("time_stream_dist.py needs a CUDA device: the hetmers path has no CPU fallback")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if "MASTER_ADDR" not in os.environ:                       # plain `python tools/time_stream_dist.py`: one rank
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29731")
    nccl = world > 1 and torch.cuda.device_count() >= world
    dev = torch.device("cuda", rank if nccl else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl" if nccl else "gloo", rank=rank, world_size=world)
    try:
        G = synth.calibrate_G(K, int(a.nels), PLOIDY, HET, COV, LCUT)
        keys, cnt = synth.synth_table(K, G, PLOIDY, HET, COV, LCUT, SEED, device=dev)
        n = keys.numel()
        ht, h_rec, h_idx = host_records(torch, dev, keys, cnt)
        del keys, cnt
        torch.cuda.empty_cache()
        L = _lib.lib()
        budget = int(a.budget_gb * 1e9)

        ref, ms_inproc, res_inproc = None, None, None
        if rank == 0:                                          # the in-process streamed call, shards on this GPU
            os.environ["HETMERS_STREAM"] = "1"
            L.hm_set_device_budget(budget)
            devs = (C.c_int * world)(*([dev.index] * world))
            ref = torch.empty(_lib.PLOT_CELLS, dtype=torch.int64, pin_memory=True)
            try:
                for i in range(max(a.warmup, 1) + a.steps):
                    if i == max(a.warmup, 1):
                        t0 = time.perf_counter()
                    _lib.check(L.hm_hetmers_host(C.byref(ht), devs, world, ref.data_ptr(), None))
                ms_inproc = (time.perf_counter() - t0) / max(a.steps, 1) * 1e3
                h = C.c_void_p()
                _lib.check(L.hm_scan_create(C.byref(ht), devs, world, C.byref(h)))
                try:
                    p2 = torch.empty(_lib.PLOT_CELLS, dtype=torch.int64)
                    _lib.check(L.hm_scan_run(h, p2.data_ptr(), None))
                    b, c = C.c_int64(), C.c_int64()
                    L.hm_scan_residency(h, C.byref(b), C.byref(c))
                    res_inproc = (b.value, c.value)
                finally:
                    L.hm_scan_destroy(h)
            finally:
                os.environ.pop("HETMERS_STREAM", None)
                L.hm_set_device_budget(0)
        dist.barrier()

        sc = hd.StreamedShardedScan(ht, device=dev, budget=budget)
        try:
            rows, plots = [], []
            for i in range(max(a.warmup, 1) + a.steps):
                tm = {}
                dist.barrier()
                t0 = time.perf_counter()
                plot = sc.scan(tm)
                tm["scan_total"] = (time.perf_counter() - t0) * 1e3
                if i >= max(a.warmup, 1):
                    rows.append(tm)
                    plots.append(plot.cpu().reshape(-1))
            peak, chunks, bud = sc.residency()
            mine = {"rank": rank, "device": str(dev), "cuts": sc.cuts[rank:rank + 2], "device_bytes": peak,
                    "budget": bud, "chunks": chunks, "stats": sc.stats, "ok": sc.symm_ok(),
                    "ms_mean": {k: sum(r.get(k, 0.0) for r in rows) / max(len(rows), 1) for k in rows[0]} if rows else {},
                    "ms_scan_total_each": [r["scan_total"] for r in rows]}
        finally:
            sc.close()
        every = [None] * world
        dist.all_gather_object(every, (mine, [bool(torch.equal(p, ref)) for p in plots] if rank == 0 else []))
        if rank == 0:
            same = all(every[0][1]) and all(r[0]["ok"] for r in every)
            line = {"metric": "ms per scan, one process per rank streaming its share, vs the in-process streamed call",
                    "unit": "ms", "workload": workload_name(1), "nels": n, "world": world,
                    "backend": "nccl" if nccl else "gloo", "steps": a.steps, "warmup": max(a.warmup, 1),
                    "gpu": torch.cuda.get_device_name(dev), "power_limit": power_limit(), "budget_bytes": budget,
                    "in_process_streamed": {"ms_per_call": ms_inproc, "device_bytes": res_inproc[0],
                                            "chunks": res_inproc[1],
                                            "note": "hm_hetmers_host: create + run + destroy; the ranks' scan() "
                                                    "excludes create"},
                    "ranks": [r[0] for r in every],
                    "parity": {"plot_ranks_vs_in_process_streamed": same, "ok": same}}
            print(json.dumps(line), flush=True)
            if not same:
                sys.stderr.write("time_stream_dist.py: a rank's plot differs from the in-process streamed plot\n")
                sys.exit(3)
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
