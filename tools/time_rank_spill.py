#!/usr/bin/env python3
"""The one-process-per-GPU streamed job with each rank's candidate records and S list resident on its device against
the same job with them in host memory (dist.StreamedShardedScan(list_host_budget=...), DESIGN.md §4c, *Lists in host
memory*, *ranks*).  --world gloo ranks share GPU 0.  The table is trimmed and symmetric, shaped like bench.py's
workload (BASELINE.json configs[1]: k = 31, diploid, het 1 %, coverage 40) at --nels entries.  Both arms stream each
rank's share in the chunks of the spilled arm's plan: the spilled arm under the largest budget whose plan leaves
the lists 1.5 B per entry (they take about 3, so they do not fit and the job refuses without a list host
budget), the resident arm under that budget plus room for the rank's whole lists.  The arms alternate after
--warmup rounds, --steps calls each; a call is
one scan() then one extract() on every rank, each timed by the wall clock on every rank (the slowest rank is
reported) and split into the phases dist.StreamedShardedScan's timings give.  Medians are reported with the spill
stats (flushes, bytes each way, rounds, partitions), the device peak and the card and power limit read in the same
run.  The plots and the lists must be equal between the arms or the run exits 3; a spilled arm that did not spill
exits 2.

    python tools/time_rank_spill.py [--world 1] [--nels 3e7] [--steps 3] [--warmup 1] [--dir /tmp]
"""
import argparse
import ctypes as C
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
from tools.time_stream import power_limit  # noqa: E402


def share_budget(lib, StreamLayout, n, k, ibyte, world, share):
    """the largest device budget whose plan for `world` shares leaves a rank's resident lists at most 1.5 B per
    entry of its share (they take about 3): the lists do not fit -> (budget, the plan's chunk)"""
    lo, hi = 1 << 20, 1 << 40
    lay = StreamLayout()
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if lib.hm_stream_plan_shards(n, k, ibyte, mid, world, C.byref(lay)) != 0 or lay.list_bytes <= 3 * share // 2:
            lo = mid
        else:
            hi = mid - 1
    lib.hm_stream_plan_shards(n, k, ibyte, lo, world, C.byref(lay))
    return lo, lay.chunk


def _rank(rank, world, port, name, a, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import numpy as np
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from smudgeplot_b200 import _lib, fastk
        from smudgeplot_b200 import dist as hd
        kt = fastk.read_ktab(name, mmap=True)
        n = kt.nels
        share = -(-n // world)
        tight, chunk = share_budget(_lib.lib(), _lib.StreamLayout, n, K, kt.ibyte, world, share)
        lists = 16 * (share // 2 + 4096) + 8 * (share + 4096)    # a rank's lists at their bound
        roomy = tight + 2 * lists
        os.environ["HETMERS_STREAM_CHUNK"] = str(chunk)
        pix = np.zeros((_lib.SMAX + 1, _lib.PLOT_W), dtype=np.uint16)
        pix[1:, 1:] = 1                                           # every pixel labelled: the whole list

        def arm(budget, cap):
            sc = hd.StreamedShardedScan(name, device="cuda:0", budget=budget, list_host_budget=cap)
            try:
                ts, te = {}, {}
                dist.barrier()
                t0 = time.perf_counter()
                plot = sc.scan(timings=ts)
                t1 = time.perf_counter()
                sst, res = dict(sc.stats), sc.residency()
                recs = sc.extract(pix, dst=0, timings=te)
                t2 = time.perf_counter()
                est = dict(sc.stats)
            finally:
                sc.close()
            r = {"ms_scan": (t1 - t0) * 1e3, "ms_extract": (t2 - t1) * 1e3, "device_peak": res[0], "budget": res[2],
                 "pass1_reused": est["pass1_reused"]}
            r.update({f"scan_{p}": v for p, v in ts.items()})
            r.update({f"extract_{p}": v for p, v in te.items()})
            for tag, st in (("scan", sst), ("extract", est)):
                sp = st["spill"]
                r.update({f"{tag}_{key}": sp[key] for key in ("spilled", "flushes", "d2h_bytes", "host_peak_bytes",
                                                              "rounds", "partitions", "h2d_bytes", "slice", "part",
                                                              "ms_flush", "ms_pass2")})
            return plot.cpu().numpy(), recs, r

        arms = {"resident": lambda: arm(roomy, None), "spilled": lambda: arm(tight, 1 << 40)}
        runs, got = {key: [] for key in arms}, {}
        for step in range(a.warmup + a.steps):
            for key, fn in arms.items():
                plot, recs, r = fn()
                got[key] = (plot, recs)
                if step >= a.warmup:
                    runs[key].append(r)
        same_plot = bool(np.array_equal(got["resident"][0], got["spilled"][0]))
        same_list = rank != 0 or got["resident"][1].tobytes() == got["spilled"][1].tobytes()
        q.put((rank, {"runs": runs, "same_plot": same_plot, "same_list": bool(same_list), "chunk": chunk,
                      "budget_resident": roomy, "budget_spilled": tight,
                      "records": len(got["spilled"][1]) if rank == 0 else None}))
    finally:
        dist.barrier()
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=1, help="gloo ranks, all on GPU 0")
    ap.add_argument("--nels", type=float, default=3e7, help="entries of the trimmed, symmetric table")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--dir", default=None, help="where the table files are written (a temporary directory)")
    a = ap.parse_args()
    import torch
    import torch.multiprocessing as mp
    if not torch.cuda.is_available():
        raise SystemExit("time_rank_spill.py needs a CUDA device: the hetmers path has no CPU fallback")
    work = tempfile.mkdtemp(prefix="time_rank_spill.", dir=a.dir)
    try:
        dev = torch.device("cuda", 0)
        G = synth.calibrate_G(K, int(a.nels), PLOIDY, HET, COV, LCUT)
        keys, cnt = synth.synth_table(K, G, PLOIDY, HET, COV, LCUT, SEED, device=dev)
        name = os.path.join(work, "t")
        kt = synth.write_table(name, K, keys, cnt, ibyte=3, nparts=4)
        n = kt.nels
        del keys, cnt, kt
        torch.cuda.empty_cache()
        ctx = mp.get_context("spawn")
        q = ctx.Queue()
        port = 38500 + os.getpid() % 2000
        procs = [ctx.Process(target=_rank, args=(r, a.world, port, name, a, q)) for r in range(a.world)]
        for p in procs:
            p.start()
        res = dict(q.get(timeout=7200) for _ in range(a.world))
        for p in procs:
            p.join(timeout=300)
        med = {}
        for key in ("resident", "spilled"):
            per_rank = [res[r]["runs"][key] for r in range(a.world)]
            fields = per_rank[0][0].keys()
            # per step: the slowest rank's value; then the median over the steps
            steps = [{f: max(per_rank[r][s][f] for r in range(a.world)) for f in fields}
                     for s in range(len(per_rank[0]))]
            med[key] = {f: sorted(s[f] for s in steps)[len(steps) // 2] for f in fields}
        same = all(res[r]["same_plot"] and res[r]["same_list"] for r in range(a.world))
        print(json.dumps({"metric": "one-process-per-GPU streamed job: lists resident against lists in host memory",
                          "unit": "ms (median over steps of the slowest rank)", "world": a.world, "nels": n, "k": K,
                          "chunk": res[0]["chunk"], "budget_resident": res[0]["budget_resident"],
                          "budget_spilled": res[0]["budget_spilled"], "records": res[0]["records"],
                          "gpu": torch.cuda.get_device_name(dev), "power_limit": power_limit(), "steps": a.steps,
                          "plots_and_lists_equal": same,
                          "ratio_scan": med["spilled"]["ms_scan"] / med["resident"]["ms_scan"],
                          "ratio_extract": med["spilled"]["ms_extract"] / med["resident"]["ms_extract"],
                          "median": med}))
        if not same:
            sys.exit(3)
        if not med["spilled"]["scan_spilled"] or med["resident"]["scan_spilled"]:
            sys.exit(2)
    finally:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
