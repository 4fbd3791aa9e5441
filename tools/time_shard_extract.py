#!/usr/bin/env python3
"""extract_kmer_pairs' list in the in-core one-process-per-GPU job (dist.ShardedScan.extract, DESIGN.md §6) on
bench.py's workload (BASELINE.json configs[1]), next to the in-core hm_scan_extract call on the same table.  The table
is written once as FastK files to a temporary directory and every rank loads its share with ShardedScan.from_ktab.
Three quarters of the plot's pixels carry a label (time_extract.label_pixels).

Per route (symm, direct) and rank: the from_ktab load, one scan(), then extract() on dst = 0 `steps` times after
`warmup` calls (the scan reused): per call the listing (kernels and their count read-backs), the D2H of the records,
and on dst the gather and the sort of every rank's records.  Prints one JSON line on rank 0 with the card name and
power limit, the records of each rank and whether each list equals the in-core list; exits 3 unless all do.
Writes nothing to the tree.

    torchrun --nproc-per-node W tools/time_shard_extract.py [--nels 2e8] [--steps 2] [--warmup 1]

Several ranks run NCCL when there is a GPU per rank, else gloo with every rank on GPU 0 (then the ranks share the
card and their collectives go through host memory).
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import COV, HET, K, LCUT, PLOIDY, SEED, workload_name  # noqa: E402
from tools import synth  # noqa: E402
from tools.time_extract import label_pixels  # noqa: E402
from tools.time_stream import power_limit  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nels", type=float, default=2e8)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    import torch
    import torch.distributed as dist
    from smudgeplot_b200 import dist as hd, fastk, hetmers
    if not torch.cuda.is_available():
        raise SystemExit("time_shard_extract.py needs a CUDA device: the hetmers path has no CPU fallback")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if "MASTER_ADDR" not in os.environ:                       # plain `python tools/time_shard_extract.py`: one rank
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29743")
    nccl = world > 1 and torch.cuda.device_count() >= world
    dev = torch.device("cuda", rank if nccl else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl" if nccl else "gloo", rank=rank, world_size=world)
    tmp = tempfile.TemporaryDirectory() if rank == 0 else None
    try:
        name = [None]
        if rank == 0:                                          # the table files (setup, untimed)
            G = synth.calibrate_G(K, int(a.nels), PLOIDY, HET, COV, LCUT)
            keys, cnt = synth.synth_table(K, G, PLOIDY, HET, COV, LCUT, SEED, device=dev)
            name[0] = os.path.join(tmp.name, "bench")
            synth.write_table(name[0], K, keys, cnt, ibyte=3, nparts=4)
            del keys, cnt
            torch.cuda.empty_cache()
        dist.broadcast_object_list(name, src=0)
        name = name[0]

        routes, lists, pix, plot = {}, [], None, None
        for route in ("symm", "direct"):
            dist.barrier()
            t0 = time.perf_counter()
            sc = hd.ShardedScan.from_ktab(name, device=dev, path=route)
            torch.cuda.synchronize(dev)
            ms_load = (time.perf_counter() - t0) * 1e3
            try:
                t0 = time.perf_counter()
                p = sc.scan().cpu().numpy().reshape(1001, 501)
                ms_scan = (time.perf_counter() - t0) * 1e3
                if pix is None:
                    plot, pix = p, label_pixels(p)
                same_plot = bool(np.array_equal(p, plot))
                rows = []
                for i in range(max(a.warmup, 1) + a.steps):
                    dist.barrier()
                    tm = {}
                    t0 = time.perf_counter()
                    recs = sc.extract(pix, dst=0, timings=tm)
                    tm["extract_total"] = (time.perf_counter() - t0) * 1e3
                    if i >= max(a.warmup, 1):
                        rows.append(tm)
                        if rank == 0:
                            lists.append((route, recs))
                st = dict(sc.stats)
                mine = {"rank": rank, "device": str(dev), "range": st["range"], "records": st["records"],
                        "slices": st["slices"], "scan_reused": st["scan_reused"], "ms_from_ktab": ms_load,
                        "ms_scan": ms_scan, "plot_equal": same_plot,
                        "ms_mean": {k: sum(r.get(k, 0.0) for r in rows) / len(rows) for k in rows[0]} if rows else {},
                        "ms_total_each": [r["extract_total"] for r in rows]}
                every = [None] * world
                dist.all_gather_object(every, mine)
                routes[route] = {"exchange": sc.exchange, "ranks": every}
            finally:
                sc.close()
        dist.barrier()

        if rank == 0:                                          # the in-core call on the same table
            with hetmers.Scan(fastk.read_ktab(name, mmap=True)) as sc:
                sc.run()
                ms_incore = []
                for i in range(max(a.warmup, 1) + a.steps):
                    t0 = time.perf_counter()
                    want = sc.extract(pix)
                    if i >= max(a.warmup, 1):
                        ms_incore.append((time.perf_counter() - t0) * 1e3)
            same = [{"route": r, "equal": bool(np.array_equal(x, want))} for r, x in lists]
            nrec = int(plot[pix > 0].sum())
            ok = all(s["equal"] for s in same) and len(want) == nrec and \
                all(rk["plot_equal"] for v in routes.values() for rk in v["ranks"])
            line = {"metric": "ms per ShardedScan.extract() after a scan (in-core, one process per GPU), vs in-core "
                              "hm_scan_extract", "unit": "ms", "workload": workload_name(1),
                    "nels": routes["symm"]["ranks"][-1]["range"][1], "world": world, "backend": "nccl" if nccl else "gloo", "steps": a.steps,
                    "warmup": max(a.warmup, 1), "gpu": torch.cuda.get_device_name(dev), "power_limit": power_limit(),
                    "records": len(want), "labelled_pixels": int((pix > 0).sum()),
                    "in_core": {"ms_per_call": ms_incore, "note": "hm_scan_extract after a run of the same scan"},
                    "routes": routes, "parity": {"lists_equal_in_core": same, "records_equal_labelled_plot":
                                                 len(want) == nrec, "ok": ok}}
            print(json.dumps(line), flush=True)
            if not ok:
                sys.stderr.write("time_shard_extract.py: a list differs from the in-core list\n")
                sys.exit(3)
    finally:
        dist.destroy_process_group()
        if tmp is not None:
            tmp.cleanup()


if __name__ == "__main__":
    main()
