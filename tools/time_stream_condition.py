#!/usr/bin/env python3
"""Scanning a raw FastK table in the one-process-per-GPU streamed job: conditioned into new table files first
(dist.condition_ktab, then StreamedShardedScan(dst).scan()) against conditioned on the way in, into host shares
(StreamedShardedScan.from_ktab(src, L=...).scan(); DESIGN.md §4f).  The table is canonical and untrimmed (counts from
1, one strand), shaped like bench.py's workload (BASELINE.json configs[1]: k = 31, diploid, het 1 %, coverage 40,
L = 12) at --nels entries, written by rank 0 to a temporary directory under --dir.  The arms alternate after
--warmup rounds; per arm the conditioning, the first scan and a second scan are timed (wall clock, every rank done),
with the peak host and device bytes; the plots must be equal or the run exits 3.  Rank 0 prints one JSON line with
the card, its power limit, the world size and the filesystem of --dir.  Run with torchrun:

    torchrun --nproc-per-node <world> tools/time_stream_condition.py [--nels 2e7] [--steps 2] [--warmup 1] [--dir /tmp]

Several ranks on a one-GPU box share device 0 (gloo); with a GPU per rank they use NCCL.
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import COV, HET, K, LCUT, PLOIDY, SEED  # noqa: E402
from tools import synth  # noqa: E402
from tools.time_condition_gpus import filesystem  # noqa: E402
from tools.time_stream import power_limit  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nels", type=float, default=2e7, help="entries of the canonical untrimmed table")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--dir", default=None, help="where the table files are written (a temporary directory)")
    a = ap.parse_args()
    import numpy as np
    import torch
    import torch.distributed as dist
    if not torch.cuda.is_available():
        raise SystemExit("time_stream_condition.py needs a CUDA device: the hetmers path has no CPU fallback")
    ngpu = torch.cuda.device_count()
    backend = "nccl" if ngpu >= int(os.environ.get("WORLD_SIZE", "1")) > 1 else "gloo"
    dist.init_process_group(backend)
    world, rank = dist.get_world_size(), dist.get_rank()
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    from smudgeplot_b200 import dist as hd
    from smudgeplot_b200 import fastk
    work = None
    try:
        if rank == 0:
            work = tempfile.mkdtemp(prefix="time_stream_condition.", dir=a.dir)
            G = synth.calibrate_G(K, int(2 * a.nels), PLOIDY, HET, COV, 1)
            keys, cnt = synth.synth_table(K, G, PLOIDY, HET, COV, 1, SEED, device=dev)
            keep = keys <= synth.revcomp_left(keys, K)                 # what FastK writes: the canonical strand
            ku = synth.keys_to_u64_numpy(keys[keep].cpu())
            cn = cnt[keep].cpu().numpy().astype(np.uint16)
            del keys, cnt, keep
            torch.cuda.empty_cache()
            fastk.write_ktab(os.path.join(work, "src"), K, ku, cn, ibyte=3, nparts=4)
            del ku, cn
        box = [work]
        dist.broadcast_object_list(box, src=0)
        work = box[0]
        src, dst = os.path.join(work, "src"), os.path.join(work, "dst")
        n = fastk.read_ktab(src).nels

        def synced(fn):
            torch.cuda.synchronize(dev)
            dist.barrier()
            t0 = time.perf_counter()
            out = fn()
            torch.cuda.synchronize(dev)
            dist.barrier()
            return out, (time.perf_counter() - t0) * 1e3

        def files():
            cst, ms_cond = synced(lambda: hd.condition_ktab(src, dst, LCUT, device=dev))
            sc, ms_open = synced(lambda: hd.StreamedShardedScan(dst, device=dev))
            try:
                plot, ms_scan = synced(sc.scan)
                _, ms_scan2 = synced(sc.scan)
                peak = sc.residency()[0]
            finally:
                sc.close()
            return plot, {"ms_condition": ms_cond + ms_open, "ms_scan": ms_scan, "ms_scan_again": ms_scan2,
                          "ms_total": ms_cond + ms_open + ms_scan, "passes": cst["passes"],
                          "condition_peak_bytes": cst["peak_bytes"], "scan_peak_bytes": peak, "host_bytes": 0,
                          "bytes_written": cst["bytes_written"]}

        def host_shares():
            sc, ms_cond = synced(lambda: hd.StreamedShardedScan.from_ktab(src, device=dev, L=LCUT))
            try:
                plot, ms_scan = synced(sc.scan)
                _, ms_scan2 = synced(sc.scan)
                st, peak = sc.stats["condition"], sc.residency()[0]
            finally:
                sc.close()
            return plot, {"ms_condition": ms_cond, "ms_scan": ms_scan, "ms_scan_again": ms_scan2,
                          "ms_total": ms_cond + ms_scan, "passes": st["passes"],
                          "condition_peak_bytes": st["peak_bytes"], "scan_peak_bytes": peak,
                          "host_bytes": st["host_bytes"], "bytes_written": 0}

        arms = {"files": files, "host_shares": host_shares}
        runs = {name: [] for name in arms}
        plots = {}
        for step in range(a.warmup + a.steps):
            for name, fn in arms.items():
                plot, r = fn()
                plots[name] = plot
                if step >= a.warmup:
                    runs[name].append(r)
        same = torch.equal(plots["files"], plots["host_shares"])
        if rank == 0:
            summary = {name: {key: sorted(r[key] for r in rs)[len(rs) // 2] for key in rs[0]}
                       for name, rs in runs.items()}
            print(json.dumps({"metric": "raw table -> streamed scan across ranks: condition into files then scan, "
                                        "against condition into host shares then scan", "unit": "ms (median)",
                              "world": world, "backend": backend, "nels": n, "k": K, "L": LCUT,
                              "gpu": torch.cuda.get_device_name(dev), "power_limit": power_limit(),
                              "filesystem": filesystem(work), "steps": a.steps, "plots_equal": same,
                              "median": summary, "runs": runs}))
        if not same:
            sys.exit(3)
    finally:
        dist.barrier()
        if rank == 0 and work is not None:
            shutil.rmtree(work, ignore_errors=True)
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
