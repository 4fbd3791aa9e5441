#!/usr/bin/env python3
"""extract_kmer_pairs' list in a job whose ranks stream their own shares of bench.py's workload (BASELINE.json
configs[1]) under a device budget (dist.StreamedShardedScan.extract, DESIGN.md §4c, *Ranks*), next to the in-core
hm_scan_extract call on the same table.  Three quarters of the plot's pixels carry a label (time_extract.label_pixels).

Per rank: extract() after a scan() (pass 1 reused), `steps` times after `warmup` calls, and once on a fresh object
(pass 1 run by extract()); per call the chunk loop (pass 1), the pixmap upload, per exchange round the routed
extraction kernel (with the grouping of its queries), the query all-to-all, the answers, the answer all-to-all and
the listing of the parked candidates with the round's records D2H, then the rank's own sort, and on dst the gather
and the sort of every rank's records.  Prints one JSON line on rank 0 with the card name and power limit; exits 3
unless every list equals the in-core list.  Writes nothing to the tree.

    torchrun --nproc-per-node W tools/time_rank_extract.py --budget-gb 1.6 [--nels 2e8] [--steps 2] [--warmup 1]

Several ranks run NCCL when there is a GPU per rank, else gloo with every rank on GPU 0 (then the budget is per
rank and the ranks share the card).
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import COV, HET, K, LCUT, PLOIDY, SEED, workload_name  # noqa: E402
from smudgeplot_b200 import _lib  # noqa: E402
from tools import synth  # noqa: E402
from tools.time_extract import extract as incore_extract, label_pixels  # noqa: E402
from tools.time_stream import host_records, power_limit  # noqa: E402


def timed_extract(sc, pix):
    tm = {}
    t0 = time.perf_counter()
    recs = sc.extract(pix, timings=tm)
    tm["extract_total"] = (time.perf_counter() - t0) * 1e3
    return recs, tm, dict(sc.stats)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--budget-gb", type=float, required=True, help="device budget of each rank (GB)")
    ap.add_argument("--nels", type=float, default=2e8)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    import torch
    import torch.distributed as dist
    from smudgeplot_b200 import dist as hd
    if not torch.cuda.is_available():
        raise SystemExit("time_rank_extract.py needs a CUDA device: the hetmers path has no CPU fallback")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if "MASTER_ADDR" not in os.environ:                       # plain `python tools/time_rank_extract.py`: one rank
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29733")
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
        budget = int(a.budget_gb * 1e9)

        sc = hd.StreamedShardedScan(ht, device=dev, budget=budget)
        try:
            plot = sc.scan().cpu().numpy()
            pix = label_pixels(plot)
            rows, lists = [], []
            for i in range(max(a.warmup, 1) + a.steps):
                dist.barrier()
                recs, tm, st = timed_extract(sc, pix)
                if i >= max(a.warmup, 1):
                    rows.append(tm)
                    lists.append(recs)
            peak, _, bud = sc.residency()
        finally:
            sc.close()
        sc = hd.StreamedShardedScan(ht, device=dev, budget=budget)
        try:
            dist.barrier()
            recs, cold, cold_st = timed_extract(sc, pix)
            lists.append(recs)
            cold_peak, chunks, _ = sc.residency()
        finally:
            sc.close()
        mean = {k: sum(r.get(k, 0.0) for r in rows) / max(len(rows), 1) for k in rows[0]} if rows else {}
        mine = {"rank": rank, "device": str(dev), "cuts": sc.cuts[rank:rank + 2], "budget": bud,
                "reused": {"ms_mean": mean, "ms_total_each": [r["extract_total"] for r in rows], "stats": st,
                           "device_bytes": peak},
                "with_pass1": {"ms": cold, "stats": cold_st, "device_bytes": cold_peak, "chunks": chunks}}
        every = [None] * world
        dist.all_gather_object(every, mine)
        dist.barrier()

        if rank == 0:                                          # the in-core call on the same table
            L = _lib.lib()
            L.hm_set_device_budget(0)                          # (the ranks' budget would stream the scan)
            devs = (C.c_int * 1)(dev.index)
            h = C.c_void_p()
            _lib.check(L.hm_scan_create(C.byref(ht), devs, 1, C.byref(h)))
            try:
                p2 = np.zeros(_lib.PLOT_CELLS, dtype=np.int64)
                _lib.check(L.hm_scan_run(h, p2.ctypes.data, None))
                t0 = time.perf_counter()
                want = incore_extract(L, h, pix)
                ms_incore = (time.perf_counter() - t0) * 1e3
            finally:
                L.hm_scan_destroy(h)
            same = [bool(np.array_equal(r, want)) for r in lists]
            nrec = int(plot[pix > 0].sum())
            ok = all(same) and len(want) == nrec
            line = {"metric": "ms per extract() of a job whose ranks stream their own shares, vs in-core hm_scan_extract",
                    "unit": "ms", "workload": workload_name(1), "nels": n, "world": world,
                    "backend": "nccl" if nccl else "gloo", "steps": a.steps, "warmup": max(a.warmup, 1),
                    "gpu": torch.cuda.get_device_name(dev), "power_limit": power_limit(), "budget_bytes": budget,
                    "records": len(want), "labelled_pixels": int((pix > 0).sum()),
                    "in_core": {"ms_per_call": ms_incore, "note": "hm_scan_extract after a run of the same scan"},
                    "ranks": every, "parity": {"lists_equal_in_core": same, "records_equal_labelled_plot":
                                               len(want) == nrec, "ok": ok}}
            print(json.dumps(line), flush=True)
            if not ok:
                sys.stderr.write("time_rank_extract.py: a list differs from the in-core list\n")
                sys.exit(3)
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
